// pfz_common.cuh -- shared helpers for libpfz.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/pfz.h"

namespace pfz {

void set_error(const char *fmt, ...);

#define PFZ_CUDA_OK(expr)                                                                   \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) {                                                            \
            pfz::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__,             \
                           cudaGetErrorString(_e));                                         \
            return 1;                                                                       \
        }                                                                                   \
    } while (0)

extern unsigned long long g_launches;   // kernels launched by this library (bench.py reports it)
#define PFZ_LAUNCH_OK()                                                                     \
    do { __atomic_fetch_add(&pfz::g_launches, 1ull, __ATOMIC_RELAXED); PFZ_CUDA_OK(cudaGetLastError()); } while (0)

#define PFZ_REQUIRE(cond, ...)                                                              \
    do {                                                                                    \
        if (!(cond)) { pfz::set_error(__VA_ARGS__); return 1; }                             \
    } while (0)

static inline cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }

constexpr unsigned FULL = 0xffffffffu;

// SMs of an H100 SXM: caps the grids of grid-stride kernels (a few resident blocks per SM)
constexpr int SM_COUNT = 132;

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ int warp_incl_scan(int v) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int o = __shfl_up_sync(FULL, v, d);
        if (lane >= d) v += o;
    }
    return v;
}

__device__ __forceinline__ double shfl_d(double v, int src) {
    return __shfl_sync(FULL, v, src);
}

// exclusive scan of int32 -> int32 on a stream; ws from pfz_scan_ws_bytes(n)
int scan_exclusive_i32(const int32_t *in, int32_t *out, int64_t n, void *ws, cudaStream_t st);

}  // namespace pfz
