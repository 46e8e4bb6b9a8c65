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

// One warp's sorted top-k list (k <= 32) under the canonical key (score desc, index asc): lane r holds rank r, the valid
// entries are a prefix (j >= 0) and lanes from k on stay empty, so the only state is the lane's (s, j); the threshold is
// lane k-1's entry once it is valid.  Every lane offers one candidate per call (cj < 0: none); one ballot finds the lanes
// that beat the threshold, and those are inserted one at a time (rank by ballot, tail shifted up by one lane), re-testing
// the rest after each insert.  Indices are distinct, so the key is a strict total order and the list is the top k of
// everything offered, whatever the order of the offers.
struct WarpTopK {
    double s; int j; int k;
    __device__ __forceinline__ static bool before(double a, int ai, double b, int bi) { return a > b || (a == b && ai < bi); }
    __device__ __forceinline__ void init(int k_) { s = 0.0; j = -1; k = k_; }
    __device__ __forceinline__ bool wants(double cs, int cj) const {
        const double ts = shfl_d(s, k - 1);
        const int tj = __shfl_sync(FULL, j, k - 1);
        return cj >= 0 && (tj < 0 || before(cs, cj, ts, tj));
    }
    __device__ __forceinline__ void offer(double cs, int cj) {
        const int lane = lane_id();
        unsigned m = __ballot_sync(FULL, wants(cs, cj));
        while (m) {
            const int src = __ffs(m) - 1;
            const double bs = shfl_d(cs, src);
            const int bj = __shfl_sync(FULL, cj, src);
            const int pos = __popc(__ballot_sync(FULL, j >= 0 && before(s, j, bs, bj)));
            const double us = __shfl_up_sync(FULL, s, 1);
            const int uj = __shfl_up_sync(FULL, j, 1);
            if (lane > pos) { s = us; j = lane < k ? uj : -1; }
            else if (lane == pos) { s = bs; j = bj; }
            m = (m & (m - 1)) & __ballot_sync(FULL, wants(cs, cj));
        }
    }
    // the row's k slots; empty slots (-1, 0.0)
    __device__ __forceinline__ void store(int32_t *idx, double *val) const {
        const int lane = lane_id();
        if (lane < k) { idx[lane] = j; val[lane] = j >= 0 ? s : 0.0; }
    }
};

// exclusive scan of int32 -> int32 on a stream; ws from pfz_scan_ws_bytes(n)
int scan_exclusive_i32(const int32_t *in, int32_t *out, int64_t n, void *ws, cudaStream_t st);

}  // namespace pfz
