// pfz_spcos.cu -- K2: sparse cosine (from CSR x to inverted index) with a fused per-row top-k, plus
// the inverted-index build and the top-k list merge.
//
// Replaces sparse_dot_topn.awesome_cossim_topn (call site polyfuzz/models/_utils.py:82) and the
// reference's Python post-processing (polyfuzz/models/_utils.py:84-91, 128-146).
//
// Layout in HBM
//   from matrix : CSR, int32 indptr/indices (ascending per row), float64 data
//   to index    : postings grouped by (term, to-tile): seg[t*n_tiles + tau] .. seg[t*n_tiles + tau + 1]
//                 post_idx int32 (to-row local to the shard), post_val float64
//   A to-tile is `tile` consecutive to-rows; one warp owns one (from-row, tile) unit at a time with a
//   private fp64 accumulator array acc[tile] in shared memory, so that
//     - the per (from-row, to-row) additions happen in ascending term order (the warp walks the
//       from-row's terms in order; inside one term every to-row occurs at most once => no conflicts),
//     - no atomics and no block barriers are needed (only __syncwarp between terms).
//   First touches are detected by acc == 0 (all weights are > 0) and recorded in a per-warp list, so
//   the selection phase visits touched to-rows only (work ~ postings, not ~ n_from * n_to).
#include <stdlib.h>
#include "pfz_common.cuh"

namespace pfz {

// ---- inverted index build ---------------------------------------------------------------------
__global__ void index_count_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices, int n_rows, int tile, int n_tiles,
                                   int32_t *__restrict__ cnt) {
    const int lane = lane_id();
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (int r = gw; r < n_rows; r += nw) {
        const int tau = r / tile;
        for (int p = indptr[r] + lane; p < indptr[r + 1]; p += 32)
            atomicAdd(&cnt[(int64_t)indices[p] * n_tiles + tau], 1);
    }
}

__global__ void index_fill_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices, const double *__restrict__ data,
                                  int n_rows, int tile, int n_tiles, const int32_t *__restrict__ seg, int32_t *__restrict__ cur,
                                  uint16_t *__restrict__ post_idx, double *__restrict__ post_val, int *__restrict__ term_maxw_bits) {
    const int lane = lane_id();
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (int r = gw; r < n_rows; r += nw) {
        const int tau = r / tile;
        for (int p = indptr[r] + lane; p < indptr[r + 1]; p += 32) {
            const int64_t c = (int64_t)indices[p] * n_tiles + tau;
            const int pos = seg[c] + atomicAdd(&cur[c], 1);
            post_idx[pos] = (uint16_t)(r - tau * tile);
            post_val[pos] = data[p];
            // per-term maximum weight, rounded up to fp32 (positive floats order like their bit patterns)
            if (term_maxw_bits) atomicMax(&term_maxw_bits[indices[p]], __float_as_int(__double2float_ru(data[p])));
        }
    }
}

// Posting order inside a (term, tile) segment is free (see pfz.h), so it is chosen for the consumer:
// K2's 32 lanes read-modify-write acc[row] as 8-byte words, i.e. two 16-lane transactions over 16
// double-wide banks.  Each segment is rearranged in "rounds" that contain every (row mod 16) residue at
// most once, residues ascending, so a 16-lane window rarely holds two rows of the same bank
// (random order: ~2.8 wavefronts per transaction; rounds: close to 1).
constexpr int BANK_ORDER_MAX = 512;     // longer segments (only with very large tiles) keep their fill order
// MOD = number of distinct shared-memory banks one accumulator word can fall into: 16 for the fp64 accumulators
// (double-wide banks), 32 for the fp32 accumulators of the mixed-precision and from-row-block kernels.
template <int MOD>
__global__ void __launch_bounds__(128) index_bank_order_kernel(const int32_t *__restrict__ seg, int64_t ncell, uint16_t *__restrict__ post_idx,
                                                               double *__restrict__ post_val) {
    __shared__ uint16_t s_idx[4][BANK_ORDER_MAX];
    __shared__ uint16_t s_rank[4][BANK_ORDER_MAX];
    __shared__ double s_val[4][BANK_ORDER_MAX];
    __shared__ int s_cnt[4][MOD];
    const int lane = lane_id(), w = threadIdx.x >> 5;
    const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t c0 = gw * 32; c0 < ncell; c0 += nw * 32) {
        // each lane inspects one cell, the warp then serves the cells that need work
        int s = 0, len = 0;
        if (c0 + lane < ncell) { s = seg[c0 + lane]; len = seg[c0 + lane + 1] - s; }
        unsigned todo = __ballot_sync(FULL, len > MOD && len <= BANK_ORDER_MAX);
        while (todo) {
            const int src = __ffs(todo) - 1; todo &= todo - 1;
            const int cs = __shfl_sync(FULL, s, src), cl = __shfl_sync(FULL, len, src);
            if (lane < MOD) s_cnt[w][lane] = 0;
            __syncwarp();
            for (int q = lane; q < cl; q += 32) {
                const uint16_t j = post_idx[cs + q];
                s_idx[w][q] = j; s_val[w][q] = post_val[cs + q];
                s_rank[w][q] = (uint16_t)atomicAdd(&s_cnt[w][j & (MOD - 1)], 1);
            }
            __syncwarp();
            int cnt[MOD];
#pragma unroll
            for (int r = 0; r < MOD; ++r) cnt[r] = s_cnt[w][r];
            for (int q = lane; q < cl; q += 32) {
                const int r = s_idx[w][q] & (MOD - 1), i = s_rank[w][q];
                int pos = 0;
#pragma unroll
                for (int r2 = 0; r2 < MOD; ++r2) pos += min(cnt[r2], i) + ((r2 < r && cnt[r2] > i) ? 1 : 0);
                post_idx[cs + pos] = s_idx[w][q];
                post_val[cs + pos] = s_val[w][q];
            }
            __syncwarp();
        }
    }
}

__global__ void to_f32_kernel(const double *__restrict__ x, int64_t n_minus, const int32_t *__restrict__ n_ptr, float *__restrict__ y) {
    const int64_t n = n_ptr ? (int64_t)*n_ptr : n_minus;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) y[i] = (float)x[i];
}

// ---- K2 --------------------------------------------------------------------------------------
// ranking key: (score desc, idx asc); "a before b"
__device__ __forceinline__ bool key_before(double sa, int ia, double sb, int ib) {
    return (sa > sb) || (sa == sb && ia < ib);
}

struct SpcosParams {
    const int32_t *a_indptr; const int32_t *a_indices; const double *a_data; int n_from;
    const int32_t *seg; const uint16_t *post_idx; const double *post_val;
    const float *post_val32; const int32_t *b_indptr; const int32_t *b_indices; const double *b_data;   // mixed-precision variant
    const float *term_maxw; float prune_alpha;      // upper-bound pruning (mixed-precision variant only; term_maxw may be NULL)
    int n_vocab, tile, n_tiles, n_to;
    int k; double min_sim; int self_match; int64_t from_base, to_base;
    int n_splits; const double *excl_val; const int32_t *excl_idx;
    int32_t *top_idx; double *top_val; int32_t *row_counter;
};

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32) spcos_list_kernel(const SpcosParams P) {
    extern __shared__ __align__(16) unsigned char dyn[];
    const int lane = lane_id();
    const int w = threadIdx.x >> 5;
    const unsigned lt = (1u << lane) - 1u;
    // per-warp arenas: acc double[tile] | touched uint16[tile]
    double *acc = reinterpret_cast<double *>(dyn) + (size_t)w * P.tile;
    uint16_t *touched = reinterpret_cast<uint16_t *>(dyn + (size_t)WARPS * P.tile * 8) + (size_t)w * P.tile;
    for (int q = lane; q < P.tile; q += 32) acc[q] = 0.0;
    __syncwarp();

    const int split = blockIdx.y;
    const int tiles_per = (P.n_tiles + P.n_splits - 1) / P.n_splits;
    const int tau_lo = split * tiles_per;
    const int tau_hi = min(P.n_tiles, tau_lo + tiles_per);
    int32_t *counter = P.row_counter + split;

    for (;;) {
        int i = 0;
        if (lane == 0) i = atomicAdd(counter, 1);
        i = __shfl_sync(FULL, i, 0);
        if (i >= P.n_from) break;

        const int a0 = P.a_indptr[i];
        const int m = P.a_indptr[i + 1] - a0;
        // top-k list: lane r holds rank r (r < k); initial entries (min_sim, -1) reject score <= min_sim
        double tv = P.min_sim; int ti = -1;
        double kv = P.min_sim; int ki = -1;             // current k-th entry (threshold)
        // exclusive lower key for paging (candidates must rank strictly after it)
        double xv = 0.0; int xi = -1; bool has_x = false;
        if (P.excl_val) { xv = P.excl_val[i]; xi = P.excl_idx[i]; has_x = xi >= 0; }
        const int64_t self_j = P.from_base + i - P.to_base;     // local to-row of the diagonal

        for (int tau = tau_lo; tau < tau_hi; ++tau) {
            int ntouched = 0;
            for (int tb = 0; tb < m; tb += 32) {
                const int kk = tb + lane;
                int s = 0, len = 0; double v = 0.0;
                if (kk < m) {
                    const int t = P.a_indices[a0 + kk];
                    v = P.a_data[a0 + kk];
                    const int64_t c = (int64_t)t * P.n_tiles + tau;
                    s = P.seg[c];
                    len = P.seg[c + 1] - s;
                }
                unsigned live = __ballot_sync(FULL, len > 0);
                while (live) {                                   // ascending lane == ascending term
                    const int src = __ffs(live) - 1; live &= live - 1;
                    const int ss = __shfl_sync(FULL, s, src);
                    const int sl = __shfl_sync(FULL, len, src);
                    const double sv = shfl_d(v, src);
                    for (int c0 = 0; c0 < sl; c0 += 32) {
                        const int q = c0 + lane;
                        bool first = false; int jl = 0;
                        if (q < sl) {
                            jl = P.post_idx[ss + q];
                            const double prod = __dmul_rn(sv, P.post_val[ss + q]);
                            const double old = acc[jl];
                            acc[jl] = __dadd_rn(old, prod);
                            first = (old == 0.0);
                        }
                        const unsigned fm = __ballot_sync(FULL, first);
                        if (first) touched[ntouched + __popc(fm & lt)] = (uint16_t)jl;
                        ntouched += __popc(fm);
                    }
                    __syncwarp();
                }
            }
            // selection over touched to-rows
            for (int c0 = 0; c0 < ntouched; c0 += 32) {
                const int q = c0 + lane;
                double sc = 0.0; int j = -1; bool cand = false;
                if (q < ntouched) {
                    const int jl = touched[q];
                    sc = acc[jl];
                    acc[jl] = 0.0;
                    const int jloc = tau * P.tile + jl;
                    j = (int)(P.to_base + jloc);
                    cand = key_before(sc, j, kv, ki);
                    if (P.self_match && (int64_t)jloc == self_j) cand = false;
                    if (has_x && !key_before(xv, xi, sc, j)) cand = false;
                }
                unsigned cm = __ballot_sync(FULL, cand);
                while (cm) {
                    const int src = __ffs(cm) - 1; cm &= cm - 1;
                    const double cs = shfl_d(sc, src);
                    const int cj = __shfl_sync(FULL, j, src);
                    if (!key_before(cs, cj, kv, ki)) continue;   // threshold may have risen meanwhile
                    // insert: position = number of list entries that stay before the candidate
                    const bool stays = (lane < P.k) && key_before(tv, ti, cs, cj);
                    const int pos = __popc(__ballot_sync(FULL, stays));
                    const double uv = __shfl_up_sync(FULL, tv, 1);
                    const int ui = __shfl_up_sync(FULL, ti, 1);
                    if (lane > pos) { tv = uv; ti = ui; }
                    else if (lane == pos) { tv = cs; ti = cj; }
                    kv = shfl_d(tv, P.k - 1);
                    ki = __shfl_sync(FULL, ti, P.k - 1);
                }
            }
            __syncwarp();
        }
        if (lane < P.k) {
            const size_t o = ((size_t)split * P.n_from + i) * P.k + lane;
            P.top_idx[o] = ti;
            P.top_val[o] = (ti >= 0) ? tv : 0.0;
        }
    }
}


// ---- K2, dense-regime variant ----------------------------------------------------------------
// Same ownership (one warp = one (from-row, to-tile) unit, private acc[tile]) but tuned for inputs
// where a from-row touches a sizeable fraction of every tile (company names: ~24 %):
//   * no touched list: a to-row becomes a candidate the moment its running sum first passes the
//     current k-th key (partial sums only grow: all weights > 0); it is flagged in a per-tile byte map
//     (rare after the first tiles) and examined with its FINAL sum at the end of the unit;
//   * acc is cleared densely with 16-byte stores (tile/64 instructions per lane);
//   * the unit's work items (<= 32 consecutive postings of one term) are written to a small table
//     first, then consumed by a branch-free loop that keeps D items' loads in flight across term
//     boundaries -- with a large tile only a dozen warps fit per SM, so memory-level parallelism has
//     to come from inside each warp.
struct __align__(16) WorkItem { int off; int cnt; double v; };

// ---- inline-PTX helpers for the dense kernel's inner loop ---------------------------------------
// Explicit 32-bit shared-window addresses and predicated instructions: the generic-pointer forms made
// the compiler re-derive the shared window base and wrap every item in convergence barriers.
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
// work item {int off; int cnt; double v} with one 16-byte load
__device__ __forceinline__ void lds_item(unsigned a, unsigned &off, int &cnt, double &v) {
    unsigned lo, hi;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(off), "=r"(cnt), "=r"(lo), "=r"(hi) : "r"(a) : "memory");
    v = __hiloint2double((int)hi, (int)lo);
}
// lanes below cnt load their posting (tile-local row, weight); the others get the dummy row / weight 0
__device__ __forceinline__ void ldg_posting(const uint16_t *pi, const double *pv, int lane, int cnt, unsigned dummy, unsigned &jl, double &w) {
    asm volatile("{ .reg .pred p; setp.lt.s32 p, %2, %3; mov.u32 %0, %4; mov.f64 %1, 0d0000000000000000;\n\t"
                 "@p ld.global.nc.u16 %0, [%5]; @p ld.global.nc.f64 %1, [%6]; }"
                 : "=&r"(jl), "=&d"(w) : "r"(lane), "r"(cnt), "r"(dummy), "l"(pi), "l"(pv) : "memory");
}
// The whole read-modify-write of one posting.  Idle lanes (row == dummy) issue no shared-memory access at
// all (a shared dummy row would cost an extra bank wavefront per half-warp).  The product is rounded
// before the add (mul.rn + add.rn are never contracted), as in the reference's scalar loop.  When the
// running sum passes thr for the first time the row's flag byte is set and `any` records it.
__device__ __forceinline__ void rmw_posting(unsigned acc_s, unsigned flags_s, unsigned row, unsigned dummy, double v, double w, double thr,
                                            unsigned &any) {
    asm volatile("{ .reg .pred p, q, r; .reg .f64 o, n, pr; .reg .b16 one; .reg .u32 a, f;\n\t"
                 "setp.ne.u32 p, %3, %4; mov.f64 o, 0d0000000000000000;\n\t"
                 "shl.b32 a, %3, 3; add.u32 a, a, %1; add.u32 f, %2, %3;\n\t"
                 "@p ld.shared.f64 o, [a];\n\t"
                 "mul.rn.f64 pr, %5, %6; add.rn.f64 n, o, pr;\n\t"
                 "@p st.shared.f64 [a], n;\n\t"
                 "setp.gt.f64 q, o, %7; setp.gt.and.f64 r, n, %7, !q; mov.b16 one, 1;\n\t"
                 "@r st.shared.u8 [f], one; selp.u32 %0, 1, %0, r; }"
                 : "+r"(any) : "r"(acc_s), "r"(flags_s), "r"(row), "r"(dummy), "d"(v), "d"(w), "d"(thr) : "memory");
}



// ---- mixed-precision filter (PFZ_K2_DENSE32) --------------------------------------------------------
// The accumulators, the posting weights and the from-row weights are fp32: half the shared-memory and L2
// bytes per posting.  The fp32 sums only FILTER: a to-row is flagged when its sum first passes
// thr - MARGIN, and every flagged row is re-scored exactly -- fp64, ascending term order, products rounded
// before the add -- by merging the two CSR rows, so the ranking and the returned scores are the canonical
// ones bit for bit.  |fp32 sum - exact| <= ~70 * 2^-24 + 3 * 2^-24 < 5e-6 for l2-normalised rows (all
// terms positive, exact sum <= 1) with ~70 terms; rows of up to 128 terms (engine.DENSE32_MAX_ROW_NNZ) stay below 7.7e-6, and the
// k-th gate compares two fp32 sums (<= 1.55e-5 combined): MARGIN = 3e-5 leaves a factor of two.
constexpr double K2_MARGIN = 3e-5;
__device__ __forceinline__ void lds_item32(unsigned a, unsigned &off, int &cnt, float &v) {
    unsigned vv;
    [[maybe_unused]] unsigned pad;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(off), "=r"(cnt), "=r"(vv), "=r"(pad) : "r"(a) : "memory");
    v = __uint_as_float(vv);
}
__device__ __forceinline__ void ldg_posting32(const uint16_t *pi, const float *pv, int lane, int cnt, unsigned dummy, unsigned &jl, float &w) {
    asm volatile("{ .reg .pred p; setp.lt.s32 p, %2, %3; mov.u32 %0, %4; mov.f32 %1, 0f00000000;\n\t"
                 "@p ld.global.nc.u16 %0, [%5]; @p ld.global.nc.f32 %1, [%6]; }"
                 : "=&r"(jl), "=&f"(w) : "r"(lane), "r"(cnt), "r"(dummy), "l"(pi), "l"(pv) : "memory");
}
__device__ __forceinline__ void rmw_posting32(unsigned acc_s, unsigned flags_s, unsigned row, unsigned dummy, float v, float w, float thr,
                                              unsigned &any) {
    asm volatile("{ .reg .pred p, q, r; .reg .f32 o, n; .reg .b16 one; .reg .u32 a, f;\n\t"
                 "setp.ne.u32 p, %3, %4; mov.f32 o, 0f00000000;\n\t"
                 "shl.b32 a, %3, 2; add.u32 a, a, %1; add.u32 f, %2, %3;\n\t"
                 "@p ld.shared.f32 o, [a];\n\t"
                 "fma.rn.f32 n, %5, %6, o;\n\t"
                 "@p st.shared.f32 [a], n;\n\t"
                 "setp.gt.f32 q, o, %7; setp.gt.and.f32 r, n, %7, !q; mov.b16 one, 1;\n\t"
                 "@r st.shared.u8 [f], one; @r add.u32 %0, %0, 1; }"
                 : "+r"(any) : "r"(acc_s), "r"(flags_s), "r"(row), "r"(dummy), "f"(v), "f"(w), "f"(thr) : "memory");
}
// canonical score of (from-row a, to-row b): common terms in ascending order, product rounded, then added
__device__ __forceinline__ double exact_dot(const int32_t *__restrict__ ai, const double *__restrict__ av, int an,
                                            const int32_t *__restrict__ bi, const double *__restrict__ bv, int bn) {
    double s = 0.0;
    int p = 0, q = 0;
    while (p < an && q < bn) {
        const int ca = ai[p], cb = bi[q];
        if (ca == cb) { s = __dadd_rn(s, __dmul_rn(av[p], bv[q])); ++p; ++q; }
        else if (ca < cb) ++p; else ++q;
    }
    return s;
}
// largest float not above x (x >= 0)
__device__ __forceinline__ float float_floor(double x) {
    float f = (float)x;
    if ((double)f > x) f = __uint_as_float(__float_as_uint(f) - 1u);
    return f;
}

// Register caps (inherited, not re-tuned on H100): the mixed-precision kernel at 64 registers (16 blocks of 2 warps per
// SM, a few spilled bytes), the fp64 kernel at 80 (12 blocks); fewer registers spill into the hot loop.
template <int WARPS, int D, bool APPROX, bool PRUNE>
__global__ void __launch_bounds__(WARPS * 32, (APPROX && !PRUNE && D <= 4) ? 16 : 12) spcos_dense_kernel(const SpcosParams P) {
    extern __shared__ __align__(16) unsigned char dyn[];
    const int lane = lane_id();
    const int w = threadIdx.x >> 5;
    const int T = P.tile;
    const int max_items = (T >> 5) + 32 + 2 * D;
    // per-warp arena: acc (double | float)[T + 4] | items WorkItem[max_items] | flags uint8[T + 16] | cand int[64]
    constexpr int ES = APPROX ? 4 : 8;
    const size_t arena = (size_t)(T + 4) * ES + (size_t)max_items * sizeof(WorkItem) + (size_t)T + 16 + 256;
    unsigned char *base = dyn + (size_t)w * ((arena + 15) & ~(size_t)15);
    double *acc = reinterpret_cast<double *>(base);
    WorkItem *items = reinterpret_cast<WorkItem *>(base + (size_t)(T + 4) * ES);
    unsigned char *flags = base + (size_t)(T + 4) * ES + (size_t)max_items * sizeof(WorkItem);
    int *cand = reinterpret_cast<int *>(flags + T + 16);           // mixed precision: flagged to-rows awaiting exact re-scoring
    for (int q = lane; q < (T + 4) * ES / 4; q += 32) reinterpret_cast<unsigned *>(base)[q] = 0u;
    for (int q = lane; q < T + 16; q += 32) flags[q] = 0;
    __syncwarp();
    const unsigned acc_s = smem_u32(acc), items_s = smem_u32(items), flags_s = smem_u32(flags);
    const uint16_t *pidx_lane = P.post_idx + lane;
    const double *pval_lane = P.post_val + lane;
    const float *pval32_lane = P.post_val32 + lane;
    asm volatile("" : "+l"(pidx_lane), "+l"(pval_lane), "+l"(pval32_lane));   // keep the base pointers in registers
    const int32_t *__restrict__ seg = P.seg;
    const int n_tiles = P.n_tiles, K = P.k;

    const int split = blockIdx.y;
    const int tiles_per = (P.n_tiles + P.n_splits - 1) / P.n_splits;
    const int tau_lo = split * tiles_per;
    const int tau_hi = min(P.n_tiles, tau_lo + tiles_per);
    const int ntau = tau_hi - tau_lo;
    int32_t *counter = P.row_counter + split;

    for (;;) {
        int i = 0;
        if (lane == 0) i = atomicAdd(counter, 1);
        i = __shfl_sync(FULL, i, 0);
        if (i >= P.n_from) break;

        const int a0 = P.a_indptr[i];
        const int m = P.a_indptr[i + 1] - a0;
        double tv = P.min_sim; int ti = -1;
        double kv = P.min_sim; int ki = -1;
        // pass(x) := x > thr encodes "the running sum ranks before the k-th key": thr = kv while the list is
        // not full (strict; untouched sums are 0) and the double just below kv once it is (inclusive: ties are
        // settled on the index at the end of the unit)
        double thr = fmax(P.min_sim, 0.0);
        float thr32 = float_floor(fmax(P.min_sim - K2_MARGIN, 0.0));     // flag threshold of the fp32 filter (see flag_thr)
        double xv = 0.0; int xi = -1; bool has_x = false;
        if (P.excl_val) { xv = P.excl_val[i]; xi = P.excl_idx[i]; has_x = xi >= 0; }
        const int64_t self_j = P.from_base + i - P.to_base;
        // start with the tile that holds the diagonal: in sorted real-world lists the best matches sit
        // near the row itself, so the k-th key is high from the first unit on (order does not affect results)
        int first_tau = tau_lo;
        if (P.self_match && self_j >= (int64_t)tau_lo * T && self_j < (int64_t)tau_hi * T) first_tau = (int)(self_j / T);

        // exact scoring + insertion of up to 32 candidates (one per lane); mixed precision batches its flagged rows
        // across units so that each round of dependent CSR loads serves a full warp
        int ncand = 0; bool need_reselect = false;
        auto score_round = [&](int n_round) {
            double sc = 0.0; int j = -1; bool cnd = false;
            if (lane < n_round) {
                const int jloc = cand[lane];
                const int b0 = P.b_indptr[jloc];
                sc = exact_dot(P.a_indices + a0, P.a_data + a0, m, P.b_indices + b0, P.b_data + b0, P.b_indptr[jloc + 1] - b0);
                j = (int)(P.to_base + jloc);
                cnd = key_before(sc, j, kv, ki);
                if (P.self_match && (int64_t)jloc == self_j) cnd = false;
                if (has_x && !key_before(xv, xi, sc, j)) cnd = false;
            }
            unsigned cm = __ballot_sync(FULL, cnd);
            while (cm) {
                const int src = __ffs(cm) - 1;
                const double cs = shfl_d(sc, src);
                const int cjx = __shfl_sync(FULL, j, src);
                const bool stays = (lane < K) && key_before(tv, ti, cs, cjx);
                const int pos = __popc(__ballot_sync(FULL, stays));
                const double uv = __shfl_up_sync(FULL, tv, 1);
                const int ui = __shfl_up_sync(FULL, ti, 1);
                if (lane > pos) { tv = uv; ti = ui; }
                else if (lane == pos) { tv = cs; ti = cjx; }
                kv = shfl_d(tv, K - 1);
                ki = __shfl_sync(FULL, ti, K - 1);
                cnd = cnd && lane != src && key_before(sc, j, kv, ki);
                cm = __ballot_sync(FULL, cnd);
            }
            need_reselect = true;
        };

        // rows with <= 32 terms (the common case) keep their terms in registers across tiles
        int t_reg = 0; double v_reg = 0.0; int prev_end = 0;
        if (m <= 32 && lane < m) { t_reg = P.a_indices[a0 + lane]; v_reg = P.a_data[a0 + lane]; }

        // Upper-bound pruning (mixed precision, rows of <= 32 terms).  Term t can add at most ub_t = v_t * max_j w_jt
        // to any score.  A set NE of terms with sum ub < alpha * (kth - MARGIN) is skipped altogether (heavy, low-idf
        // n-grams such as "inc": long posting lists, tiny contributions); the flag threshold drops by that sum, so
        // every to-row that could still reach the k-th key is flagged by its remaining terms and scored exactly from
        // the CSR rows (which include the skipped terms).  Re-selected whenever the k-th key has moved.
        bool skip_term = false; float ub_ne = 0.f;
        float ub_k = 0.f; int df_k = 0;
        const bool prune = PRUNE && APPROX && P.term_maxw != nullptr && m <= 32 && P.prune_alpha > 0.f;
        if (prune && lane < m) {
            ub_k = __fmul_ru(__double2float_ru(v_reg), P.term_maxw[t_reg]);
            df_k = seg[(int64_t)(t_reg + 1) * n_tiles] - seg[(int64_t)t_reg * n_tiles];
        }
        auto select_ne = [&]() {
            skip_term = false; ub_ne = 0.f;
            if (!prune) return;
            float budget = P.prune_alpha * fmaxf((float)(kv - K2_MARGIN), 0.f);
            if (ki < 0) budget = 0.f;                               // list not full: every touched row is a candidate
            for (int r = 0; r < 8; ++r) {                           // up to 8 terms, longest posting list first
                int best = (lane < m && !skip_term && ub_k <= budget && df_k > 0) ? df_k : -1;
                int who = lane;
#pragma unroll
                for (int d = 16; d; d >>= 1) {
                    const int ob = __shfl_xor_sync(FULL, best, d), ow = __shfl_xor_sync(FULL, who, d);
                    if (ob > best || (ob == best && ow < who)) { best = ob; who = ow; }
                }
                if (best < 0) break;
                const float u = __shfl_sync(FULL, ub_k, who);
                if (lane == who) skip_term = true;
                ub_ne = __fadd_ru(ub_ne, u); budget -= u;
            }
        };
        if (PRUNE) select_ne();
        auto flag_thr = [&]() { return float_floor(fmax(fmax(kv - K2_MARGIN, 0.0) - (double)ub_ne, 0.0)); };

        for (int it = 0; it < ntau; ++it) {
            int tau = first_tau + it; if (tau >= tau_hi) tau -= ntau;
            bool any_post = false; unsigned crossed_any = 0u;
            if (APPROX && need_reselect) { if (PRUNE) select_ne(); thr32 = flag_thr(); need_reselect = false; }
            for (int tb = 0; tb < m; tb += 32) {
                const int kk = tb + lane;
                int s = 0, len = 0; double v = 0.0;
                if (kk < m) {
                    int t;
                    if (m <= 32) { t = t_reg; v = v_reg; } else { t = P.a_indices[a0 + kk]; v = P.a_data[a0 + kk]; }
                    const int64_t c = (int64_t)t * n_tiles + tau;
                    const int e = seg[c + 1];
                    s = (m <= 32 && it > 0 && tau != tau_lo) ? prev_end : seg[c];
                    prev_end = e;
                    len = (PRUNE && skip_term) ? 0 : e - s;
                }
                // work-item table: lane k appends its ceil(len/32) items at the exclusive prefix of the counts.
                // A to-row may occur under several terms, so a term group can need more items than the table
                // holds (cap >= one term's worth): it is then consumed in batches of whole terms, in order.
                const int nch = (len + 31) >> 5;
                const int incl = warp_incl_scan(nch);
                const int n_total = __shfl_sync(FULL, incl, 31);
                if (n_total == 0) continue;
                any_post = true;
                const int cap = (T >> 5) + 32;
                for (int start = 0; start < n_total;) {
                    const bool inb = nch > 0 && incl - nch >= start && incl <= start + cap;
                    const unsigned bm = __ballot_sync(FULL, inb);
                    const int endv = __shfl_sync(FULL, incl, 31 - __clz(bm));
                    const int N = endv - start;
                    if (inb) {
                        int o = incl - nch - start, so = s, rem = len;
                        const double vitem = APPROX ? __hiloint2double(0, (int)__float_as_uint((float)v)) : v;   // fp32 weight in the low word
                        while (rem > 0) { WorkItem wi; wi.off = so; wi.cnt = rem; wi.v = vitem; items[o] = wi; ++o; so += 32; rem -= 32; }
                    }
                    if (lane < 2 * D) { WorkItem wi; wi.off = 0; wi.cnt = 0; wi.v = 0.0; items[N + lane] = wi; }   // padding
                    __syncwarp();
                    // branch-free consumer: slot d holds item b+d; after it is consumed the slot is refilled with
                    // item b+d+D (padding items have cnt = 0, so no guard is needed).  Idle lanes add 0 to the dummy
                    // row T.  No warp barrier between items: the loop body has no branch, the warp stays converged
                    // and its shared-memory instructions complete in program order.
                    if (!APPROX) {
                        unsigned rj[D]; double rw[D], rv[D];
#pragma unroll
                        for (int d = 0; d < D; ++d) {
                            unsigned off; int cnt;
                            lds_item(items_s + d * 16, off, cnt, rv[d]);
                            ldg_posting(pidx_lane + off, pval_lane + off, lane, cnt, (unsigned)T, rj[d], rw[d]);
                        }
                        unsigned it_s = items_s + D * 16;
                        for (int b = 0; b < N; b += D) {
#pragma unroll
                            for (int d = 0; d < D; ++d) {
                                rmw_posting(acc_s, flags_s, rj[d], (unsigned)T, rv[d], rw[d], thr, crossed_any);
                                unsigned off; int cnt;
                                lds_item(it_s + d * 16, off, cnt, rv[d]);
                                ldg_posting(pidx_lane + off, pval_lane + off, lane, cnt, (unsigned)T, rj[d], rw[d]);
                            }
                            it_s += D * 16;
                        }
                    } else {
                        unsigned rj[D]; float rw[D], rv[D];
#pragma unroll
                        for (int d = 0; d < D; ++d) {
                            unsigned off; int cnt;
                            lds_item32(items_s + d * 16, off, cnt, rv[d]);
                            ldg_posting32(pidx_lane + off, pval32_lane + off, lane, cnt, (unsigned)T, rj[d], rw[d]);
                        }
                        unsigned it_s = items_s + D * 16;
                        for (int b = 0; b < N; b += D) {
#pragma unroll
                            for (int d = 0; d < D; ++d) {
                                rmw_posting32(acc_s, flags_s, rj[d], (unsigned)T, rv[d], rw[d], thr32, crossed_any);
                                unsigned off; int cnt;
                                lds_item32(it_s + d * 16, off, cnt, rv[d]);
                                ldg_posting32(pidx_lane + off, pval32_lane + off, lane, cnt, (unsigned)T, rj[d], rw[d]);
                            }
                            it_s += D * 16;
                        }
                    }
                    __syncwarp();
                    start = endv;
                }
            }
            if (!any_post) continue;
            // candidates: flagged to-rows -> final sums -> exact key test -> insertion
            if (__any_sync(FULL, crossed_any != 0u)) {
                // Mixed precision only: when many rows are flagged (the first units of a from-row, before the
                // k-th key has risen) re-scoring all of them exactly would dominate.  Pass A finds the k-th largest
                // fp32 sum among the flagged rows (shared memory only); a row can reach the unit's exact top-k only
                // if its fp32 sum is within MARGIN of that value, so pass B re-scores just those.
                float gate = thr32;
                if (APPROX) {
                    const int nflag = (int)__reduce_add_sync(FULL, crossed_any);   // each lane counted its own flags (rmw_posting32)
                    if (nflag > 2 * K + 32 && !has_x) {              // (paging excludes rows by exact key: no pre-selection then)
                        const float *acc32 = reinterpret_cast<const float *>(acc);
                        float lv = -1.f;                                  // lane r: r-th largest fp32 sum so far (r < K)
                        float kth = -1.f;
                        for (int w0 = 0; w0 < T; w0 += 128) {
                            const int q4 = w0 + lane * 4;
                            unsigned bits = (q4 < T) ? *reinterpret_cast<const unsigned *>(flags + q4) : 0u;
                            while (__ballot_sync(FULL, bits != 0u)) {
                                float a = -2.f;
                                if (bits) {
                                    const int b8 = (__ffs(bits) - 1) >> 3; bits &= ~(0xffu << (b8 * 8)); a = acc32[q4 + b8];
                                    if (P.self_match && (int64_t)(tau * T + q4 + b8) == self_j) a = -2.f;     // the diagonal never competes
                                }
                                unsigned cm = __ballot_sync(FULL, a > kth);
                                while (cm) {
                                    const int src = __ffs(cm) - 1;
                                    const float ca = __shfl_sync(FULL, a, src);
                                    const int pos = __popc(__ballot_sync(FULL, (lane < K) && lv >= ca));
                                    const float up = __shfl_up_sync(FULL, lv, 1);
                                    if (lane > pos) lv = up; else if (lane == pos) lv = ca;
                                    kth = __shfl_sync(FULL, lv, K - 1);
                                    a = (lane == src) ? -2.f : a;
                                    cm = __ballot_sync(FULL, a > kth);
                                }
                            }
                        }
                        gate = fmaxf(gate, float_floor(fmax((double)kth - K2_MARGIN - (double)ub_ne, 0.0)));
                    }
                }
                for (int w00 = 0; w00 < T; w00 += 512) {            // 16 flag bytes per lane per step; empty 512-row spans cost one vote
                  uint4 fb = make_uint4(0u, 0u, 0u, 0u);
                  const int q16 = w00 + lane * 16;
                  if (q16 < T) {
                      fb = *reinterpret_cast<const uint4 *>(flags + q16);
                      if (fb.x | fb.y | fb.z | fb.w) *reinterpret_cast<uint4 *>(flags + q16) = make_uint4(0u, 0u, 0u, 0u);
                  }
                  if (!__any_sync(FULL, (fb.x | fb.y | fb.z | fb.w) != 0u)) continue;
#pragma unroll
                  for (int wsel = 0; wsel < 4; ++wsel) {
                    unsigned bits = wsel == 0 ? fb.x : wsel == 1 ? fb.y : wsel == 2 ? fb.z : fb.w;
                    const int q4 = q16 + wsel * 4;
                    while (__ballot_sync(FULL, bits != 0u)) {
                        if (APPROX) {
                            bool take = false; int jloc = 0;
                            if (bits) {
                                const int b8 = (__ffs(bits) - 1) >> 3; bits &= ~(0xffu << (b8 * 8));
                                const int jl = q4 + b8;
                                jloc = tau * T + jl;
                                take = reinterpret_cast<const float *>(acc)[jl] > gate;
                            }
                            const unsigned tm = __ballot_sync(FULL, take);
                            if (take) cand[ncand + __popc(tm & ((1u << lane) - 1u))] = jloc;
                            ncand += __popc(tm);
                            __syncwarp();
                            if (ncand >= 32) {                        // a full warp of candidates: score them now
                                score_round(32);
                                __syncwarp();
                                const int rest = ncand - 32;
                                int mv = 0;
                                if (lane < rest) mv = cand[32 + lane];
                                __syncwarp();
                                if (lane < rest) cand[lane] = mv;
                                ncand = rest;
                                __syncwarp();
                            }
                            continue;
                        }
                        double sc = 0.0; int j = -1; bool cnd = false;
                        if (bits) {
                            const int b8 = (__ffs(bits) - 1) >> 3; bits &= ~(0xffu << (b8 * 8));
                            const int jl = q4 + b8;
                            const int jloc = tau * T + jl;
                            sc = acc[jl];
                            j = (int)(P.to_base + jloc);
                            cnd = key_before(sc, j, kv, ki);
                            if (P.self_match && (int64_t)jloc == self_j) cnd = false;
                            if (has_x && !key_before(xv, xi, sc, j)) cnd = false;
                        }
                        unsigned cm = __ballot_sync(FULL, cnd);
                        while (cm) {
                            const int src = __ffs(cm) - 1;
                            const double cs = shfl_d(sc, src);
                            const int cjx = __shfl_sync(FULL, j, src);
                            const bool stays = (lane < K) && key_before(tv, ti, cs, cjx);
                            const int pos = __popc(__ballot_sync(FULL, stays));
                            const double uv = __shfl_up_sync(FULL, tv, 1);
                            const int ui = __shfl_up_sync(FULL, ti, 1);
                            if (lane > pos) { tv = uv; ti = ui; }
                            else if (lane == pos) { tv = cs; ti = cjx; }
                            kv = shfl_d(tv, K - 1);
                            ki = __shfl_sync(FULL, ti, K - 1);
                            // prune: drop the inserted lane and everything the new k-th key now rejects
                            cnd = cnd && lane != src && key_before(sc, j, kv, ki);
                            cm = __ballot_sync(FULL, cnd);
                        }
                    }
                  }
                }
                thr = (ki >= 0) ? __longlong_as_double(__double_as_longlong(kv) - 1) : fmax(kv, 0.0);
            }
            __syncwarp();
            // dense clear, 16 B per lane per store
            {
                double2 *a2 = reinterpret_cast<double2 *>(acc);
                const double2 z = make_double2(0.0, 0.0);
                for (int q = lane; q < (T * ES >> 4); q += 32) a2[q] = z;
            }
            __syncwarp();
        }
        if (APPROX && ncand > 0) { __syncwarp(); score_round(ncand); __syncwarp(); }       // leftovers (ncand < 32)
        if (lane < K) {
            const size_t o = ((size_t)split * P.n_from + i) * K + lane;
            P.top_idx[o] = ti;
            P.top_val[o] = (ti >= 0) ? tv : 0.0;
        }
    }
}

// merge: one warp per row; lists are individually sorted but that is not relied upon
__global__ void __launch_bounds__(256) topk_merge_kernel(const int32_t *__restrict__ idx, const double *__restrict__ val, int n_lists, int n_from,
                                                         int k_in, int k_out, int32_t *__restrict__ out_idx, double *__restrict__ out_val) {
    const int lane = lane_id();
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (int i = gw; i < n_from; i += nw) {
        double tv = 0.0; int ti = -1;       // sentinel entries: idx -1 ranks after everything valid
        double kv = 0.0; int ki = -1; bool full = false;
        int filled = 0;
        for (int l = 0; l < n_lists; ++l) {
            const size_t b = ((size_t)l * n_from + i) * k_in;
            for (int c0 = 0; c0 < k_in; c0 += 32) {
                const int q = c0 + lane;
                double sc = 0.0; int j = -1;
                if (q < k_in) { j = idx[b + q]; sc = val[b + q]; }
                unsigned cm = __ballot_sync(FULL, j >= 0);
                while (cm) {
                    const int src = __ffs(cm) - 1; cm &= cm - 1;
                    const double cs = shfl_d(sc, src);
                    const int cj = __shfl_sync(FULL, j, src);
                    if (full && !key_before(cs, cj, kv, ki)) continue;
                    const bool stays = (lane < filled) && key_before(tv, ti, cs, cj);
                    const int pos = __popc(__ballot_sync(FULL, stays));
                    const double uv = __shfl_up_sync(FULL, tv, 1);
                    const int ui = __shfl_up_sync(FULL, ti, 1);
                    if (lane > pos) { tv = uv; ti = ui; }
                    else if (lane == pos) { tv = cs; ti = cj; }
                    if (filled < k_out) ++filled;
                    full = filled == k_out;
                    kv = shfl_d(tv, k_out - 1);
                    ki = __shfl_sync(FULL, ti, k_out - 1);
                }
            }
        }
        if (lane < k_out) {
            const bool ok = lane < filled;
            out_idx[(size_t)i * k_out + lane] = ok ? ti : -1;
            out_val[(size_t)i * k_out + lane] = ok ? tv : 0.0;
        }
    }
}

static int grid_for2(int64_t work_items, int threads, int cap) {
    int64_t g = (work_items + threads - 1) / threads;
    if (g < 1) g = 1;
    if (g > cap) g = cap;
    return (int)g;
}

}  // namespace pfz

using namespace pfz;

extern "C" {

int pfz_index_build(const int32_t *indptr, const int32_t *indices, const double *data, int32_t n_rows, int32_t n_vocab, int32_t tile,
                    int32_t n_tiles, int32_t flags, int32_t *seg, uint16_t *post_idx, double *post_val, float *post_val32, float *term_maxw,
                    void *ws, void *stream) {
    PFZ_REQUIRE(tile > 0 && tile <= 65536, "pfz_index_build: tile %d out of range (1..65536)", tile);
    PFZ_REQUIRE((int64_t)n_tiles * tile >= n_rows, "pfz_index_build: n_tiles*tile < n_rows");
    const int64_t ncell = (int64_t)n_vocab * n_tiles;
    PFZ_REQUIRE(ncell + 1 < (1ll << 31), "pfz_index_build: n_vocab*n_tiles = %lld too large", (long long)ncell);
    cudaStream_t st = as_stream(stream);
    // ws layout: cur int32[ncell+1] | scan ws
    int32_t *cur = reinterpret_cast<int32_t *>(ws);
    void *sws = reinterpret_cast<char *>(ws) + ((((size_t)ncell + 1) * 4 + 255) / 256) * 256;
    PFZ_CUDA_OK(cudaMemsetAsync(seg, 0, ((size_t)ncell + 1) * 4, st));
    if (n_rows > 0) {
        index_count_kernel<<<grid_for2((int64_t)n_rows * 32, 256, SM_COUNT * 16), 256, 0, st>>>(indptr, indices, n_rows, tile, n_tiles, seg);
        PFZ_LAUNCH_OK();
    }
    if (scan_exclusive_i32(seg, seg, ncell + 1, sws, st)) return 1;
    if (n_rows > 0) {
        PFZ_CUDA_OK(cudaMemsetAsync(cur, 0, ((size_t)ncell + 1) * 4, st));
        if (term_maxw) PFZ_CUDA_OK(cudaMemsetAsync(term_maxw, 0, (size_t)n_vocab * 4, st));
        index_fill_kernel<<<grid_for2((int64_t)n_rows * 32, 256, SM_COUNT * 16), 256, 0, st>>>(indptr, indices, data, n_rows, tile, n_tiles, seg, cur,
                                                                                            post_idx, post_val, reinterpret_cast<int *>(term_maxw));
        PFZ_LAUNCH_OK();
        if (flags & PFZ_INDEX_BANK_ORDER32) {
            index_bank_order_kernel<32><<<grid_for2(ncell, 128, SM_COUNT * 16), 128, 0, st>>>(seg, ncell, post_idx, post_val);
            PFZ_LAUNCH_OK();
        } else if (flags & PFZ_INDEX_BANK_ORDER) {
            index_bank_order_kernel<16><<<grid_for2(ncell, 128, SM_COUNT * 16), 128, 0, st>>>(seg, ncell, post_idx, post_val);
            PFZ_LAUNCH_OK();
        }
        if (post_val32) {                                       // fp32 copy of the weights for the mixed-precision filter
            to_f32_kernel<<<SM_COUNT * 8, 256, 0, st>>>(post_val, 0, seg + ncell, post_val32);
            PFZ_LAUNCH_OK();
        }
    }
    return 0;
}

int pfz_spcos_topk(const int32_t *a_indptr, const int32_t *a_indices, const double *a_data, int32_t n_from, const int32_t *seg,
                   const uint16_t *post_idx, const double *post_val, const float *post_val32, const int32_t *b_indptr,
                   const int32_t *b_indices, const double *b_data, const float *term_maxw, int32_t n_vocab, int32_t tile, int32_t n_tiles, int32_t n_to, int32_t k,
                   double min_similarity, int32_t self_match, int64_t from_index_base, int64_t to_index_base, int32_t n_splits,
                   const double *excl_val, const int32_t *excl_idx, int32_t *top_idx, double *top_val, int32_t *row_counter,
                   int32_t variant, void *stream) {
    PFZ_REQUIRE(k >= 1 && k <= 32, "pfz_spcos_topk: k=%d unsupported (1..32 per call; page with excl_* for more)", k);
    PFZ_REQUIRE(tile > 0 && tile <= 65536 && (tile % 64) == 0, "pfz_spcos_topk: tile %d must be a multiple of 64 in 64..65536", tile);
    PFZ_REQUIRE(n_splits >= 1 && n_splits <= n_tiles, "pfz_spcos_topk: n_splits %d out of range", n_splits);
    PFZ_REQUIRE(variant == PFZ_K2_LIST || variant == PFZ_K2_DENSE || variant == PFZ_K2_DENSE32, "pfz_spcos_topk: unknown variant %d", variant);
    PFZ_REQUIRE(variant != PFZ_K2_DENSE32 || (post_val32 && b_indptr && b_indices && b_data),
                "pfz_spcos_topk: PFZ_K2_DENSE32 needs post_val32 and the to-matrix CSR");
    if (n_from <= 0) return 0;
    cudaStream_t st = as_stream(stream);
    int dev = 0, sms = 0, smem_max = 0;
    PFZ_CUDA_OK(cudaGetDevice(&dev));
    PFZ_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    PFZ_CUDA_OK(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    PFZ_CUDA_OK(cudaMemsetAsync(row_counter, 0, sizeof(int32_t) * (size_t)n_splits, st));
    const char *env_a = getenv("PFZ_K2_PRUNE_ALPHA");            // developer knob; 0 disables upper-bound pruning
    const float prune_alpha = env_a ? (float)atof(env_a) : 0.0f; // measured slower on the benchmark data: off by default
    SpcosParams P{a_indptr, a_indices, a_data, n_from, seg, post_idx, post_val, post_val32, b_indptr, b_indices, b_data, term_maxw, prune_alpha,
                  n_vocab, tile, n_tiles, n_to, k, min_similarity, self_match,
                  from_index_base, to_index_base, n_splits, excl_val, excl_idx, top_idx, top_val, row_counter};
    auto launch = [&](auto kernel, int warps, size_t smem) -> int {
        PFZ_REQUIRE(smem <= (size_t)smem_max, "pfz_spcos_topk: tile %d needs %zu B shared memory > %d available", tile, smem, smem_max);
        PFZ_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int occ = 0;
        PFZ_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, warps * 32, smem));
        if (occ < 1) occ = 1;
        int gx = sms * occ;
        const int need = (n_from + warps - 1) / warps;
        if (gx > need) gx = need;
        if (n_splits > 1) { gx = (gx + n_splits - 1) / n_splits; if (gx < 1) gx = 1; }
        kernel<<<dim3(gx, n_splits), warps * 32, smem, st>>>(P);
        PFZ_LAUNCH_OK();
        return 0;
    };
    if (variant == PFZ_K2_LIST) {
        constexpr int WARPS = 8;
        return launch(spcos_list_kernel<WARPS>, WARPS, (size_t)WARPS * tile * 10);
    }
    constexpr int WARPS = 2;
    const int es = variant == PFZ_K2_DENSE32 ? 4 : 8;
    auto arena_of = [&](int D) { return (((size_t)(tile + 4) * es + (size_t)((tile >> 5) + 32 + 2 * D) * sizeof(WorkItem) + (size_t)tile + 16 + 256) + 15) & ~(size_t)15; };
    const char *env_d = getenv("PFZ_K2_DEPTH");                  // developer knob (pipeline depth); default 4
    const int depth = env_d ? atoi(env_d) : 4;
    if (variant == PFZ_K2_DENSE32) {
        if (prune_alpha > 0.f && term_maxw) return launch(spcos_dense_kernel<WARPS, 4, true, true>, WARPS, (size_t)WARPS * arena_of(4));
        if (depth == 8) return launch(spcos_dense_kernel<WARPS, 8, true, false>, WARPS, (size_t)WARPS * arena_of(8));
        if (depth == 6) return launch(spcos_dense_kernel<WARPS, 6, true, false>, WARPS, (size_t)WARPS * arena_of(6));
        if (depth == 3) return launch(spcos_dense_kernel<WARPS, 3, true, false>, WARPS, (size_t)WARPS * arena_of(3));
        if (depth == 2) return launch(spcos_dense_kernel<WARPS, 2, true, false>, WARPS, (size_t)WARPS * arena_of(2));
        return launch(spcos_dense_kernel<WARPS, 4, true, false>, WARPS, (size_t)WARPS * arena_of(4));
    }
    if (depth == 8) return launch(spcos_dense_kernel<WARPS, 8, false, false>, WARPS, (size_t)WARPS * arena_of(8));
    return launch(spcos_dense_kernel<WARPS, 4, false, false>, WARPS, (size_t)WARPS * arena_of(4));
}

int pfz_topk_merge(const int32_t *idx, const double *val, int32_t n_lists, int32_t n_from, int32_t k_in, int32_t k_out, int32_t *out_idx,
                   double *out_val, void *stream) {
    PFZ_REQUIRE(k_out >= 1 && k_out <= 32, "pfz_topk_merge: k_out=%d unsupported (1..32)", k_out);
    PFZ_REQUIRE(n_lists >= 1 && k_in >= 1, "pfz_topk_merge: bad n_lists/k_in");
    if (n_from <= 0) return 0;
    topk_merge_kernel<<<grid_for2((int64_t)n_from * 32, 256, SM_COUNT * 16), 256, 0, as_stream(stream)>>>(idx, val, n_lists, n_from, k_in, k_out, out_idx, out_val);
    PFZ_LAUNCH_OK();
    return 0;
}
}
