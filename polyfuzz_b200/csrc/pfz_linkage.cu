// pfz_linkage.cu -- K7: single linkage (polyfuzz/linkage.py:25-51) on the device.
// The reference walks the kept rows in order with a dict m and a counter c = 0:
//     if not m.get(F): (if not m.get(T): m[T] = m[F] = c; c += 1  else: m[F] = m[T])
// Cluster id 0 is falsy, so the first kept row r0 writes 0 and every later test treats its keys as unset.  A value, once
// nonzero, never changes, so row p's outcome depends only on which of its keys are nonzero before it, and key x is nonzero
// before p iff a kept row q in (r0, p) has F_q = x or is a create with T_q = x (DESIGN.md 4.13 states and proves the rule):
//
//   static   r0 = the first kept row; firstF[x] = min{q > r0 : F_q = x}; pend[x] = min{q > r0 : T_q = x}   (atomicMin)
//   rounds   every undecided row p reads firstF, createMin (creates decided so far) and pend (the first row with T = x that
//            was undecided at the end of the previous round): F known set -> skip; F known unset and T known set -> inherit;
//            both known unset -> create.  The first undecided row always decides, so every round makes progress.  LK_ROUNDS
//            rounds are enqueued back to back, each returning at once when the device count of undecided rows is zero
//   finish   one warp decides whatever is left in row order (nothing when the count is zero)
//   ids      create ids = exclusive scan of the create flags; an inherit row takes the value of the row that first made its T
//            nonzero, min(firstF[T], createMin[T]), resolved by pointer jumping; each key's first write is (row, slot), a create
//            writing T (slot 0) before F (slot 1), and a scan over the 2n slots gives the insertion ranks
//   groups   each cluster's first key (from its create row's two keys and r0's), the representative key of every key, and a
//            stable radix sort of the keys in insertion order by their cluster's first rank: the reference's `clusters`
//
// Only min-reductions and integer sums go through atomics, so the outputs do not depend on thread scheduling; a round may see
// a create decided by another thread of the same round, which is a true fact and only lets it decide earlier.
#include <algorithm>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include "pfz_common.cuh"

namespace pfz {

constexpr int LK_THREADS = 256;
constexpr int32_t LK_INF = 0x7F7F7F7F;      // memset(0x7F) writes it; above every row index and slot code (n < 2^30)
constexpr int LK_ROUNDS = 12;               // real top-1 self-matches take 4-7 rounds (DESIGN.md 4.13)
constexpr int LK_MAX_JUMPS = 32;
enum : int32_t { LK_NONE = 0, LK_UNDEC = 1, LK_SKIP = 2, LK_INHERIT = 3, LK_CREATE = 4 };

static int lk_grid(int64_t items) {
    int64_t g = (items + LK_THREADS - 1) / LK_THREADS;
    if (g > SM_COUNT * 8) g = SM_COUNT * 8;
    return g < 1 ? 1 : (int)g;
}

#define LK_LOOP(i, count) for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (count); i += (int64_t)gridDim.x * blockDim.x)

// one atomic per warp for a per-thread sum or minimum
__device__ __forceinline__ void warp_add(int32_t *dst, int v) {
    v = __reduce_add_sync(FULL, v);
    if (lane_id() == 0 && v) atomicAdd(dst, v);
}
__device__ __forceinline__ void warp_min(int32_t *dst, int v) {
    v = __reduce_min_sync(FULL, v);
    if (lane_id() == 0 && v < LK_INF) atomicMin(dst, v);
}

// status[p] = undecided for a kept row (Similarity > min_similarity; NaN fails, as in pandas), none otherwise; r0 = first kept row
__global__ void __launch_bounds__(LK_THREADS) lk_kept_kernel(const double *__restrict__ sim, double thr, int32_t n,
                                                            int32_t *__restrict__ status, int32_t *r0) {
    int32_t first = LK_INF;
    LK_LOOP(p, n) {
        const bool kept = sim == nullptr || sim[p] > thr;
        status[p] = kept ? LK_UNDEC : LK_NONE;
        if (kept && p < first) first = (int32_t)p;
    }
    warp_min(r0, first);
}

__global__ void __launch_bounds__(LK_THREADS) lk_static_kernel(const int32_t *__restrict__ F, const int32_t *__restrict__ T, int32_t n,
                                                              int32_t *__restrict__ status, const int32_t *__restrict__ r0p,
                                                              int32_t *firstF, int32_t *pend0, int32_t *count0) {
    const int32_t r0 = *r0p;
    int c = 0;
    LK_LOOP(p, n) {
        if (status[p] != LK_UNDEC) continue;
        if (p == r0) { status[p] = LK_CREATE; continue; }
        atomicMin(&firstF[F[p]], (int32_t)p);
        atomicMin(&pend0[T[p]], (int32_t)p);
        ++c;
    }
    warp_add(count0, c);
}

// One round.  cur: first row per T key undecided at the end of the previous round; nxt: the same for this round (filled here);
// clr: the buffer the next round fills, read by the previous round, reset here.
__global__ void __launch_bounds__(LK_THREADS) lk_round_kernel(const int32_t *__restrict__ F, const int32_t *__restrict__ T, int32_t n,
                                                             int32_t n_keys, int32_t *__restrict__ status, const int32_t *__restrict__ firstF,
                                                             int32_t *createMin, const int32_t *__restrict__ cur, int32_t *nxt,
                                                             int32_t *__restrict__ clr, const int32_t *__restrict__ count_in,
                                                             int32_t *count_out, int32_t *umin_out) {
    if (*count_in == 0) return;
    int c = 0;
    int32_t um = LK_INF;
    LK_LOOP(i, (int64_t)max(n, n_keys)) {
        if (i < n_keys) clr[i] = LK_INF;
        if (i < n && status[i] == LK_UNDEC) {
            const int32_t p = (int32_t)i, f = F[p], t = T[p];
            int32_t out = LK_UNDEC;
            if (firstF[f] < p || createMin[f] < p) out = LK_SKIP;
            else if (cur[f] >= p) {                                          // no row before p can still make F nonzero
                if (firstF[t] < p || createMin[t] < p) out = LK_INHERIT;
                else if (cur[t] >= p) out = LK_CREATE;
            }
            if (out != LK_UNDEC) {
                status[p] = out;
                if (out == LK_CREATE) atomicMin(&createMin[t], p);
            } else {
                atomicMin(&nxt[t], p);
                ++c;
                um = min(um, p);
            }
        }
    }
    warp_add(count_out, c);
    warp_min(umin_out, um);
}

// The rows left after the rounds, in row order by one warp: every earlier row is decided when a row's turn comes.
__global__ void lk_finish_kernel(const int32_t *__restrict__ F, const int32_t *__restrict__ T, int32_t n, int32_t *status,
                                 const int32_t *__restrict__ firstF, int32_t *createMin, const int32_t *__restrict__ count_in,
                                 const int32_t *__restrict__ umin) {
    if (*count_in == 0) return;
    const int lane = lane_id();
    for (int32_t b = *umin & ~31; b < n; b += 32) {
        const int32_t p = b + lane;
        const bool und = p < n && status[p] == LK_UNDEC;
        unsigned m = __ballot_sync(FULL, und);
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            if (lane == src) {
                const int32_t f = F[p], t = T[p];
                int32_t out;
                if (firstF[f] < p || createMin[f] < p) out = LK_SKIP;
                else if (firstF[t] < p || createMin[t] < p) out = LK_INHERIT;
                else { out = LK_CREATE; if (createMin[t] > p) createMin[t] = p; }
                status[p] = out;
            }
            __syncwarp();                                                    // the write is seen by the next lane's decision
        }
    }
}

// cid[p] = 1 for a create row (scanned in place into the create ids), cid[n] = 0
__global__ void __launch_bounds__(LK_THREADS) lk_create_flags_kernel(const int32_t *__restrict__ status, int32_t n, int32_t *__restrict__ cid) {
    LK_LOOP(p, (int64_t)n + 1) cid[p] = p < n && status[p] == LK_CREATE;
}

// ptr[p] = the row that first made T_p nonzero for an inherit row (a create or an inherit row before p), p itself otherwise
__global__ void __launch_bounds__(LK_THREADS) lk_ptr_init_kernel(const int32_t *__restrict__ T, int32_t n, const int32_t *__restrict__ status,
                                                                const int32_t *__restrict__ firstF, const int32_t *__restrict__ createMin,
                                                                int32_t *__restrict__ ptr, int32_t *count0) {
    int c = 0;
    LK_LOOP(p, n) {
        int32_t q = (int32_t)p;
        if (status[p] == LK_INHERIT) {
            const int32_t t = T[p];
            q = min(firstF[t], createMin[t]);
            c += status[q] != LK_CREATE;
        }
        ptr[p] = q;
    }
    warp_add(count0, c);
}

// ptr[p] = ptr[ptr[p]] until it reaches a create row.  A concurrent update only hands p a further ancestor, so after j launches
// every pointer is at least 2^j rows up its chain or at its create row.
__global__ void __launch_bounds__(LK_THREADS) lk_jump_kernel(int32_t n, const int32_t *__restrict__ status, int32_t *ptr,
                                                            const int32_t *__restrict__ count_in, int32_t *count_out) {
    if (*count_in == 0) return;
    int c = 0;
    LK_LOOP(p, n) {
        if (status[p] != LK_INHERIT) continue;
        int32_t q = ptr[p];
        if (status[q] == LK_CREATE) continue;
        q = ptr[q];
        ptr[p] = q;
        c += status[q] != LK_CREATE;
    }
    warp_add(count_out, c);
}

// Per key: the final value (its first nonzero writer's, 0 when only r0 wrote it, -1 when unwritten) and its first write's
// slot code 2*row + slot, recorded as slot[code] = key.
__global__ void __launch_bounds__(LK_THREADS) lk_keys_kernel(const int32_t *__restrict__ F, const int32_t *__restrict__ T, int32_t n,
                                                            int32_t n_keys, const int32_t *__restrict__ r0p, const int32_t *__restrict__ firstF,
                                                            const int32_t *__restrict__ createMin, const int32_t *__restrict__ cid,
                                                            const int32_t *__restrict__ ptr, int32_t *__restrict__ val, int32_t *__restrict__ slot) {
    const int32_t r0 = *r0p;
    const int32_t t0 = r0 < n ? T[r0] : -1, f0 = r0 < n ? F[r0] : -1;
    LK_LOOP(x, n_keys) {
        const int32_t s = min(firstF[x], createMin[x]);
        int64_t code = -1;
        if (x == t0) code = 2 * (int64_t)r0;
        else if (x == f0) code = 2 * (int64_t)r0 + 1;
        else if (s < LK_INF) code = 2 * (int64_t)s + (createMin[x] == s ? 0 : 1);
        val[x] = s < LK_INF ? cid[ptr[s]] : (code >= 0 ? 0 : -1);
        if (code >= 0) slot[code] = (int32_t)x;
    }
}

__global__ void __launch_bounds__(LK_THREADS) lk_slot_flags_kernel(const int32_t *__restrict__ slot, int64_t n_slots, int32_t *__restrict__ pos) {
    LK_LOOP(i, n_slots + 1) pos[i] = i < n_slots && slot[i] >= 0;
}

__global__ void __launch_bounds__(LK_THREADS) lk_rank_kernel(const int32_t *__restrict__ slot, int64_t n_slots, const int32_t *__restrict__ pos,
                                                            int32_t *__restrict__ rank, int32_t *__restrict__ order, int32_t *__restrict__ n_written) {
    LK_LOOP(i, n_slots) {
        const int32_t x = slot[i];
        if (x >= 0) { rank[x] = pos[i]; order[pos[i]] = x; }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *n_written = pos[n_slots];
}

// The first key (lowest rank) of each cluster.  Cluster v's keys are its create row's T and F, keys first written after that
// row by inherits, and r0's two keys when their final value is v, so only those four can come first.
__global__ void __launch_bounds__(LK_THREADS) lk_first_rank_kernel(const int32_t *__restrict__ F, const int32_t *__restrict__ T, int32_t n,
                                                                  const int32_t *__restrict__ status, const int32_t *__restrict__ r0p,
                                                                  const int32_t *__restrict__ cid, const int32_t *__restrict__ val,
                                                                  const int32_t *__restrict__ rank, int32_t *__restrict__ first_rank) {
    const int32_t r0 = *r0p;
    LK_LOOP(p, n) {
        if (status[p] != LK_CREATE) continue;
        const int32_t v = cid[p];
        const int32_t keys[4] = {T[p], F[p], T[r0], F[r0]};
        int32_t fr = LK_INF;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (val[keys[k]] == v) fr = min(fr, rank[keys[k]]);
        first_rank[v] = fr;
    }
}

// rep[x] = the first key of x's cluster; the sort input: keys in insertion order keyed by their cluster's first rank, and the
// sentinel n_keys (above every rank) past the written keys
__global__ void __launch_bounds__(LK_THREADS) lk_rep_kernel(int32_t n_keys, const int32_t *__restrict__ val, const int32_t *__restrict__ rank,
                                                           const int32_t *__restrict__ order, const int32_t *__restrict__ first_rank,
                                                           const int32_t *__restrict__ n_written, int32_t *__restrict__ rep,
                                                           int32_t *__restrict__ skey, int32_t *__restrict__ sval) {
    const int32_t nw = *n_written;
    LK_LOOP(x, n_keys) {
        const int32_t r = rank[x];
        if (r >= 0) {
            const int32_t fr = first_rank[val[x]];
            rep[x] = order[fr];
            skey[r] = fr;
            sval[r] = (int32_t)x;
        } else {
            rep[x] = -1;
        }
        if (x >= nw) { skey[x] = n_keys; sval[x] = -1; }
    }
}

// the workspace: int32 arrays at 256-byte boundaries, then CUB's temporary storage
struct LkWs {
    int32_t *inf_block;                 // firstF, createMin, pend[3], r0, umin[LK_ROUNDS + 1], first_rank[n + 1]: memset 0x7F
    int32_t *firstF, *createMin, *pend, *r0, *umin, *first_rank;
    int32_t *counts;                    // round counts [LK_ROUNDS + 1], jump counts [LK_MAX_JUMPS + 1]: memset 0
    int32_t *status, *cid, *ptr, *slot, *pos, *order, *skey, *skey_out, *sval;
    void *cub;
    size_t inf_ints, count_ints, cub_bytes, total;
};

static size_t lk_cub_bytes(int32_t n, int32_t n_keys) {
    size_t a = 0, b = 0, c = 0;
    if (cub::DeviceScan::ExclusiveSum(nullptr, a, (int32_t *)nullptr, (int64_t)n + 1) != cudaSuccess) return 0;
    if (cub::DeviceScan::ExclusiveSum(nullptr, b, (int32_t *)nullptr, 2 * (int64_t)n + 1) != cudaSuccess) return 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, c, (const int32_t *)nullptr, (int32_t *)nullptr, (const int32_t *)nullptr,
                                        (int32_t *)nullptr, (int64_t)n_keys) != cudaSuccess) return 0;
    return std::max(a, std::max(b, c));
}

static LkWs lk_carve(void *base, int32_t n, int32_t n_keys) {
    LkWs w{};
    size_t off = 0;
    char *b = (char *)base;
    auto take = [&](size_t ints) { int32_t *p = (int32_t *)(b ? b + off : nullptr); off += (ints * 4 + 255) & ~(size_t)255; return p; };
    const size_t K = (size_t)n_keys, N = (size_t)n;
    w.inf_ints = 5 * K + 1 + (LK_ROUNDS + 1) + N + 1;
    w.inf_block = take(w.inf_ints);
    if (b) {
        w.firstF = w.inf_block; w.createMin = w.firstF + K; w.pend = w.createMin + K; w.r0 = w.pend + 3 * K;
        w.umin = w.r0 + 1; w.first_rank = w.umin + LK_ROUNDS + 1;
    }
    w.count_ints = LK_ROUNDS + 1 + LK_MAX_JUMPS + 1;
    w.counts = take(w.count_ints);
    w.status = take(N); w.cid = take(N + 1); w.ptr = take(N);
    w.slot = take(2 * N); w.pos = take(2 * N + 1);
    w.order = take(K); w.skey = take(K); w.skey_out = take(K); w.sval = take(K);
    w.cub_bytes = lk_cub_bytes(n, n_keys);
    w.cub = b ? b + off : nullptr;
    off += w.cub_bytes;
    w.total = off;
    return w;
}

static int bit_length(int64_t v) { int b = 0; while (v > 0) { ++b; v >>= 1; } return b; }

}  // namespace pfz

using namespace pfz;

extern "C" {

int64_t pfz_linkage_ws_bytes(int32_t n, int32_t n_keys) {
    if (n < 0 || n >= (1 << 30) || n_keys < 0) return -1;
    return (int64_t)lk_carve(nullptr, n, n_keys).total;
}

int pfz_linkage(const int32_t *F, const int32_t *T, int32_t n, const double *similarity, double min_similarity, int32_t n_keys,
                int32_t *val, int32_t *rank, int32_t *rep, int32_t *grouped, int32_t *n_written, void *ws, int64_t ws_bytes, void *stream) {
    PFZ_REQUIRE(n >= 0 && n < (1 << 30) && n_keys >= 0 && (n == 0 || n_keys > 0),
                "pfz_linkage: n (%d) must be in [0, 2^30) and n_keys (%d) positive when n > 0", n, n_keys);
    cudaStream_t st = as_stream(stream);
    if (n == 0) {
        PFZ_CUDA_OK(cudaMemsetAsync(n_written, 0, sizeof(int32_t), st));
        return 0;
    }
    LkWs w = lk_carve(ws, n, n_keys);
    PFZ_REQUIRE(w.cub_bytes > 0 && ws_bytes >= (int64_t)w.total, "pfz_linkage: ws_bytes (%lld) below pfz_linkage_ws_bytes (%lld)",
                (long long)ws_bytes, (long long)w.total);
    const int64_t n_slots = 2 * (int64_t)n;
    PFZ_CUDA_OK(cudaMemsetAsync(w.inf_block, 0x7F, sizeof(int32_t) * w.inf_ints, st));
    PFZ_CUDA_OK(cudaMemsetAsync(w.counts, 0, sizeof(int32_t) * w.count_ints, st));
    PFZ_CUDA_OK(cudaMemsetAsync(w.slot, 0xFF, sizeof(int32_t) * (size_t)n_slots, st));
    PFZ_CUDA_OK(cudaMemsetAsync(rank, 0xFF, sizeof(int32_t) * (size_t)n_keys, st));
    const int gn = lk_grid(n), gk = lk_grid(n_keys), gnk = lk_grid(std::max(n, n_keys));
    int32_t *rounds = w.counts, *jumps = w.counts + LK_ROUNDS + 1;

    lk_kept_kernel<<<gn, LK_THREADS, 0, st>>>(similarity, min_similarity, n, w.status, w.r0);
    PFZ_LAUNCH_OK();
    lk_static_kernel<<<gn, LK_THREADS, 0, st>>>(F, T, n, w.status, w.r0, w.firstF, w.pend, rounds);
    PFZ_LAUNCH_OK();
    for (int r = 0; r < LK_ROUNDS; ++r) {
        int32_t *cur = w.pend + (size_t)(r % 3) * n_keys, *nxt = w.pend + (size_t)((r + 1) % 3) * n_keys,
                *clr = w.pend + (size_t)((r + 2) % 3) * n_keys;
        lk_round_kernel<<<gnk, LK_THREADS, 0, st>>>(F, T, n, n_keys, w.status, w.firstF, w.createMin, cur, nxt, clr, rounds + r,
                                                    rounds + r + 1, w.umin + r + 1);
        PFZ_LAUNCH_OK();
    }
    lk_finish_kernel<<<1, 32, 0, st>>>(F, T, n, w.status, w.firstF, w.createMin, rounds + LK_ROUNDS, w.umin + LK_ROUNDS);
    PFZ_LAUNCH_OK();

    size_t bytes = w.cub_bytes;
    lk_create_flags_kernel<<<gn, LK_THREADS, 0, st>>>(w.status, n, w.cid);
    PFZ_LAUNCH_OK();
    PFZ_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.cub, bytes, w.cid, (int64_t)n + 1, st));
    lk_ptr_init_kernel<<<gn, LK_THREADS, 0, st>>>(T, n, w.status, w.firstF, w.createMin, w.ptr, jumps);
    PFZ_LAUNCH_OK();
    const int n_jumps = std::min(LK_MAX_JUMPS, bit_length(n));          // pointer chains are shorter than n rows
    for (int j = 0; j < n_jumps; ++j) {
        lk_jump_kernel<<<gn, LK_THREADS, 0, st>>>(n, w.status, w.ptr, jumps + j, jumps + j + 1);
        PFZ_LAUNCH_OK();
    }
    lk_keys_kernel<<<gk, LK_THREADS, 0, st>>>(F, T, n, n_keys, w.r0, w.firstF, w.createMin, w.cid, w.ptr, val, w.slot);
    PFZ_LAUNCH_OK();
    lk_slot_flags_kernel<<<lk_grid(n_slots + 1), LK_THREADS, 0, st>>>(w.slot, n_slots, w.pos);
    PFZ_LAUNCH_OK();
    bytes = w.cub_bytes;
    PFZ_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.cub, bytes, w.pos, n_slots + 1, st));
    lk_rank_kernel<<<lk_grid(n_slots), LK_THREADS, 0, st>>>(w.slot, n_slots, w.pos, rank, w.order, n_written);
    PFZ_LAUNCH_OK();
    lk_first_rank_kernel<<<gn, LK_THREADS, 0, st>>>(F, T, n, w.status, w.r0, w.cid, val, rank, w.first_rank);
    PFZ_LAUNCH_OK();
    lk_rep_kernel<<<gk, LK_THREADS, 0, st>>>(n_keys, val, rank, w.order, w.first_rank, n_written, rep, w.skey, w.sval);
    PFZ_LAUNCH_OK();
    bytes = w.cub_bytes;
    PFZ_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.cub, bytes, w.skey, w.skey_out, w.sval, grouped, (int64_t)n_keys, 0,
                                                bit_length(n_keys), st));
    return 0;
}
}
