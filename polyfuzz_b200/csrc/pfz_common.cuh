// pfz_common.cuh -- shared helpers for libpfz.so (sm_90a only), among them the row driver of K3 and K3b: split_groups,
// claim_row (claim_row_cta and merge_cta for one CTA per row), build_peq, the WarpTopK / WarpArgBest epilogues, start_rows and
// launch_rows / launch_ctas.
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

// One warp's arg-best under WarpTopK's key: each lane keeps the best (s, j) it was offered (cj < 0: none) and, with DIST, the
// distance that came with it; store() reduces the warp in a butterfly (the first maximal score = the lowest index among the
// maxima) and lane 0 writes the row's slot (-1, 0.0, -1 when empty).
template <bool DIST = true>
struct WarpArgBest {
    double s; int j; int d;
    __device__ __forceinline__ void init() { s = 0.0; j = -1; d = -1; }
    __device__ __forceinline__ void offer(double cs, int cj, int cd = -1) {
        if (cj >= 0 && (j < 0 || WarpTopK::before(cs, cj, s, j))) { s = cs; j = cj; if constexpr (DIST) d = cd; }
    }
    __device__ __forceinline__ void store(int32_t *idx, double *val, int32_t *dist) {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const double os = shfl_d(s, lane_id() ^ o);
            const int oj = __shfl_xor_sync(FULL, j, o);
            offer(os, oj, DIST ? __shfl_xor_sync(FULL, d, o) : -1);
        }
        if (lane_id() == 0) {
            *idx = j; *val = j >= 0 ? s : 0.0;
            if constexpr (DIST) *dist = d;
        }
    }
};

// ---- K3 / K3b row driver: one warp per from-row, the to-list in groups of 32 split over blockIdx.y ----------------------------
// the to-groups [lo, hi) of this block's split
struct GroupRange { int lo, hi; };
__device__ __forceinline__ GroupRange split_groups(int n_to, int n_splits) {
    const int n_grp = (n_to + 31) >> 5;
    const int per = (n_grp + n_splits - 1) / n_splits;
    const int lo = blockIdx.y * per;
    return {lo, min(n_grp, lo + per)};
}

// ---- the row driver's to-source: every to-string (CAND = false) or a candidate list per from-row (CAND = true) -----------
// A row is walked in steps [lo, hi) of 32 to-strings, one per lane.  All-pairs: step g is to-group g of the block's split and
// lane l takes sorted position 32g + l.  Candidate mode: step t is candidates 32t .. 32t + 31 of the row's list and lane l
// takes cand[i][32t + l] (-1: nothing to score), found at sorted position pos_of[j] (the inverse of the layout's `order`),
// i.e. group p / 32, lane p % 32 of the same packed layout.  One list per row, so candidate mode has one split.
struct CandList {
    const int32_t *idx;                 // int32 [n_from][c] to-indices (distinct per row), -1 = empty slot
    int c;                              // list length per row
    const int32_t *pos_of;              // int32 [n_to] sorted position of each to-index
};

template <bool CAND>
__device__ __forceinline__ GroupRange to_steps(int n_to, int n_splits, const CandList &cl) {
    if constexpr (CAND) return {0, (cl.c + 31) >> 5};
    else return split_groups(n_to, n_splits);
}

// the sorted position p the lane scores at step s of row i; to_have(p) tells whether there is one (all-pairs: p < n_to,
// candidate mode: p >= 0)
template <bool CAND>
__device__ __forceinline__ int to_pos(int s, int i, const CandList &cl) {
    if constexpr (CAND) {
        const int q = s * 32 + lane_id();
        const int j = q < cl.c ? cl.idx[(size_t)i * cl.c + q] : -1;
        return j >= 0 ? cl.pos_of[j] : -1;
    } else {
        return s * 32 + lane_id();
    }
}
template <bool CAND>
__device__ __forceinline__ bool to_have(int p, int n_to) { return CAND ? p >= 0 : p < n_to; }

// The lane's packed column (lane-strided words) in the layout (packed, grp_word_off) at step s for sorted position p.  A lane
// with nothing to score in candidate mode gets the layout's first column and length 0.  The warp-uniform text loops read up
// to the warp's longest string in every lane; that stays inside `packed` in candidate mode too, because groups are in
// ascending length order, so no group ends closer to the buffer's end than the longest string's words.
template <bool CAND>
__device__ __forceinline__ const uint32_t *to_column(const uint32_t *packed, const int64_t *grp_word_off, int s, int p) {
    if constexpr (CAND) return p >= 0 ? packed + grp_word_off[p >> 5] + (p & 31) : packed + lane_id();
    else return packed + grp_word_off[s] + lane_id();
}

// the warp's next from-row (from_ids[q], q from the split's counter), or -1 once all n_ids rows are taken
__device__ __forceinline__ int claim_row(int32_t *counter, const int32_t *from_ids, int n_ids) {
    int q = 0;
    if (lane_id() == 0) q = atomicAdd(counter, 1);
    q = __shfl_sync(FULL, q, 0);
    return q < n_ids ? from_ids[q] : -1;
}

// ---- CTA-per-row variant (K3b's 8- and 16-word classes): the CTA's warps share one from-row and its match masks, and warp w
// takes the split's to-groups lo + w, lo + w + warps, ...
// the CTA's next from-row, or -1; the leading barrier keeps the previous row's shared state (masks, slot, merge buffers) alive
// until every warp is done with it
__device__ __forceinline__ int claim_row_cta(int32_t *counter, const int32_t *from_ids, int n_ids, int *slot) {
    __syncthreads();
    if (threadIdx.x == 0) *slot = atomicAdd(counter, 1);
    __syncthreads();
    const int q = *slot;
    return q < n_ids ? from_ids[q] : -1;
}

// Merge the warps' WarpArgBest<false> or WarpTopK epilogues of one row: every lane leaves its (s, j) in sh_s / sh_j
// [warps * 32], and warp 0 offers the other warps' entries lane by lane to its own epilogue.  Both keys are strict total
// orders over distinct indices, so the result is that of one warp offered everything.  Returns true in warp 0, which then
// stores the row's slot(s) as the one-warp layout does.
template <typename Epi>
__device__ __forceinline__ bool merge_cta(Epi &e, double *sh_s, int *sh_j) {
    const int lane = lane_id(), w = threadIdx.x >> 5;
    sh_s[threadIdx.x] = e.s; sh_j[threadIdx.x] = e.j;
    __syncthreads();
    if (w != 0) return false;
    for (int v = 1; v < (int)(blockDim.x >> 5); ++v) e.offer(sh_s[v * 32 + lane], sh_j[v * 32 + lane]);
    return true;
}

// One warp's (CTA = false) or the whole CTA's (CTA = true) match masks: peq[sym * NW + block] bit p is set where pattern symbol
// p is sym.  cps: the m code points, mapped by sym_table (symbol 0, the text-only code points, matches nothing); pat (optional)
// receives the symbols 1-based.
template <typename W, int NW, bool CTA = false>
__device__ __forceinline__ void build_peq(W *peq, const uint32_t *cps, int m, const uint8_t *sym_table, uint8_t *pat = nullptr) {
    constexpr int B = 8 * sizeof(W);
    const int t0 = CTA ? (int)threadIdx.x : lane_id(), nt = CTA ? (int)blockDim.x : 32;
    for (int e = t0; e < 256 * NW; e += nt) peq[e] = 0;
    if constexpr (CTA) __syncthreads(); else __syncwarp();
    for (int p = t0; p < m; p += nt) {
        const uint32_t c = cps[p];
        const int s = c < 0x110000u ? sym_table[c] : 0;
        if (pat) pat[p + 1] = (uint8_t)s;
        if (s) {
            if (sizeof(W) == 8) atomicOr(reinterpret_cast<unsigned long long *>(&peq[s * NW + p / B]), 1ull << (p % B));
            else atomicOr(reinterpret_cast<unsigned *>(&peq[s * NW + p / B]), 1u << (p % B));
        }
    }
    if constexpr (CTA) __syncthreads(); else __syncwarp();
}

// warps per CTA (4, 2 or 1) for a kernel whose warps each take per_warp bytes of shared memory, within budget bytes per CTA
constexpr int warps_within(size_t per_warp, size_t budget) { return per_warp * 4 <= budget ? 4 : per_warp * 2 <= budget ? 2 : 1; }

// SM count of the current device, and the per-split row counters zeroed on st
static inline int start_rows(int32_t *counter, int n_splits, cudaStream_t st, int *sms) {
    int dev = 0;
    PFZ_CUDA_OK(cudaGetDevice(&dev));
    PFZ_CUDA_OK(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
    PFZ_CUDA_OK(cudaMemsetAsync(counter, 0, sizeof(int32_t) * (size_t)n_splits, st));
    return 0;
}

// Launch a row-driver kernel on (gx, n_splits) CTAs of `warps` warps: as many CTAs per split as fit the SMs at once, and no
// more than max_ctas (the CTAs the rows can keep busy).
template <typename Kernel, typename... Args>
static int launch_ctas(Kernel kernel, int warps, size_t smem, int max_ctas, int n_splits, int sms, cudaStream_t st, const Args &...args) {
    PFZ_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    PFZ_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, warps * 32, smem));
    if (occ < 1) occ = 1;
    int gx = sms * occ;
    if (gx > max_ctas) gx = max_ctas;
    if (gx < 1) gx = 1;
    kernel<<<dim3(gx, n_splits), warps * 32, smem, st>>>(args...);
    PFZ_LAUNCH_OK();
    return 0;
}
// one warp per row: n_ids rows keep (n_ids + warps - 1) / warps CTAs busy
template <typename Kernel, typename... Args>
static int launch_rows(Kernel kernel, int warps, size_t smem, int n_ids, int n_splits, int sms, cudaStream_t st, const Args &...args) {
    return launch_ctas(kernel, warps, smem, (n_ids + warps - 1) / warps, n_splits, sms, st, args...);
}

// exclusive scan of int32 -> int32 on a stream; ws from pfz_scan_ws_bytes(n)
int scan_exclusive_i32(const int32_t *in, int32_t *out, int64_t n, void *ws, cudaStream_t st);

}  // namespace pfz
