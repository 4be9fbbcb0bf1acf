// Shared helpers for the fastmot_b200 C-ABI library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>

#define FM_OK 0
#define FM_ERR_CUDA 1
#define FM_ERR_ARG 2
#define FM_ERR_CAPACITY 3

extern "C" void fm_set_last_error(const char* msg);

extern "C" void fm_count_launches(int n);

#define FM_CHECK_LAUNCH(name)                                                      \
    do {                                                                           \
        fm_count_launches(1);                                                      \
        cudaError_t e__ = cudaGetLastError();                                      \
        if (e__ != cudaSuccess) {                                                  \
            char buf__[256];                                                       \
            snprintf(buf__, sizeof buf__, "%s: %s", name, cudaGetErrorString(e__)); \
            fm_set_last_error(buf__);                                              \
            return FM_ERR_CUDA;                                                    \
        }                                                                          \
    } while (0)

#define FM_REQUIRE(cond, msg)                  \
    do {                                       \
        if (!(cond)) {                         \
            fm_set_last_error(msg);            \
            return FM_ERR_ARG;                 \
        }                                      \
    } while (0)

static inline int fm_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

#define FM_NUM_SMS 132            // H100 SXM

// ---- programmatic dependent launch (PDL) -------------------------------------------------------------------------
// The conv stacks are chains of short kernels; with PDL the next kernel's CTAs are scheduled (and run their
// input-independent prologue: barrier init, index plan, weight staging) while the previous kernel's last
// wave drains.  Protocol, kept the same in every kernel launched through fm_launch_pdl:
//   * fm_pdl_trigger() first thing in the CTA (the dependent grid may be scheduled once every CTA of this grid runs),
//   * fm_pdl_wait() unconditionally, before the first access to memory another kernel produces or consumes; it
//     returns only when the preceding grid has completed and flushed, so ordering stays transitive along the stream.
__device__ __forceinline__ void fm_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void fm_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t fm_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                                        Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// round-half-to-even of a double to an integral double (matches Python/Numba round(x, 0)).
__host__ __device__ __forceinline__ double fm_rint(double x) {
#ifdef __CUDA_ARCH__
    return rint(x);
#else
    return nearbyint(x);
#endif
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
