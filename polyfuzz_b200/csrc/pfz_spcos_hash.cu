// pfz_spcos_hash.cu -- K2, SPARSE-regime variant (PFZ_K2_HASH): sparse cosine + fused per-row top-k where one CTA
// accumulates ONE from-row's postings in a shared-memory hash table keyed by the to-row.
//
// Replaces sparse_dot_topn.awesome_cossim_topn (call site polyfuzz/models/_utils.py:82) like the other K2 variants;
// bit-identical results (exact fp64 re-scoring of the candidates, canonical ranking key).
//
// Why: on sparse inputs (BASELINE configs[4]: uniform 8..32-character strings, 0.006 postings per scored pair) a from-row
// touches ~6 000 of 1 000 000 to-rows.  The tile-based kernels pay per (from-row, to-tile) unit -- 1 954 tiles x 17
// segment look-ups per row for a handful of postings each.
// Here the work is proportional to the postings: the index is tiled as coarsely as its 16-bit local rows allow (65 536 rows),
// the CTA walks the row's (term, tile) segments once, and every posting is one hash insert (atom.shared.cas) plus one
// fire-and-forget fixed-point add (red.shared.add.u32, unit 2^-26, see pfz_spcos_block.cu).  The table then is scanned
// once: sums above the row's threshold are re-scored exactly from the two CSR rows and inserted into the top-k list.
// A row whose postings exceed half the table is processed in several passes over disjoint tile ranges; a pass whose table
// still fills is redone over halved to-row ranges, so the table size is a performance knob only.
#include <stdlib.h>
#include "pfz_common.cuh"

namespace pfz {

constexpr double K2H_SCALE = 67108864.0;         // 2^26
constexpr double K2H_MARGIN = 2e-5;              // >= 2 x (1.5 units x 256 terms x 2^-26) = 1.15e-5
constexpr unsigned K2H_MARGIN_Q = 1343u;         // ceil(K2H_MARGIN * 2^26)
#ifndef PFZ_HASH_WARPS
#define PFZ_HASH_WARPS 4
#endif
constexpr int HASH_WARPS = PFZ_HASH_WARPS, HASH_NT = HASH_WARPS * 32;   // warps per CTA (= per from-row): 4 -> 8 CTAs per SM at 64 registers
constexpr int HASH_TERM_CAP = 256;               // terms per from-row
constexpr int HASH_ITEM_CAP = 128;
constexpr int HASH_CQ = 384;                     // candidate queue
constexpr unsigned HASH_EMPTY = 0xffffffffu;

struct __align__(16) HItem { int off; int cnt; unsigned keybase; unsigned v; };

struct HashParams {
    const int32_t *a_indptr; const int32_t *a_indices; const double *a_data; int n_from;
    const int32_t *seg; const uint2 *post_pk;
    const int32_t *b_indptr; const int32_t *b_indices; const double *b_data;
    int tile, n_tiles, n_to, k; double min_sim; int self_match; int64_t from_base, to_base; int n_splits;
    const double *excl_val; const int32_t *excl_idx;
    int32_t *top_idx; double *top_val; int32_t *counter; int32_t *err_flag;
};

__device__ __forceinline__ bool h_key_before(double sa, int ia, double sb, int ib) { return (sa > sb) || (sa == sb && ia < ib); }
// canonical score of (from-row a, to-row b): common terms in ascending order, product rounded, then added.  The to-row is
// staged 32 entries at a time with INDEPENDENT loads (one memory latency per chunk instead of one per merge step -- the merge
// itself chases pointers), then merged against the from-row.
__device__ __noinline__ double h_exact_dot(const int32_t *__restrict__ ai, const double *__restrict__ av, int an,
                                  const int32_t *__restrict__ bi, const double *__restrict__ bv, int bn) {
    double s = 0.0;
    int p = 0;
    for (int c0 = 0; c0 < bn && p < an; c0 += 32) {
        int ci[32]; double cv[32];                          // local memory (dynamically indexed): registers stay with the hot loop
        const int nc = min(32, bn - c0);
#pragma unroll 8
        for (int q = 0; q < nc; ++q) { ci[q] = bi[c0 + q]; cv[q] = bv[c0 + q]; }
#pragma unroll 1
        for (int q = 0; q < nc; ++q) {
            const int cb = ci[q];
            while (p < an && ai[p] < cb) ++p;
            if (p < an && ai[p] == cb) { s = __dadd_rn(s, __dmul_rn(av[p], cv[q])); ++p; }
        }
    }
    return s;
}
__device__ __forceinline__ unsigned h_thr_q(double x) {
    const double y = (x - K2H_MARGIN) * K2H_SCALE;
    return y <= 0.0 ? 0u : (unsigned)__double2ll_rd(y);
}
__device__ __forceinline__ unsigned h_sort_desc(unsigned x, int lane) {
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
            const unsigned o = __shfl_xor_sync(FULL, x, j);
            const bool keep_max = ((lane & j) == 0) == ((lane & k) == 0);
            x = keep_max ? max(x, o) : min(x, o);
        }
    }
    return x;
}

template <int H>
__host__ __device__ inline size_t hash_arena_bytes() {
    return (size_t)H * 8 + (size_t)HASH_ITEM_CAP * 16 + (size_t)HASH_TERM_CAP * 8 + (size_t)HASH_CQ * 12 + 512;
}

#ifndef PFZ_HASH_MIN_CTAS
#define PFZ_HASH_MIN_CTAS 8    // 64 registers per thread: without the bound ptxas spends 119 and only 4 CTAs fit
#endif
template <int H, int LOGH>
__global__ void __launch_bounds__(HASH_NT, PFZ_HASH_MIN_CTAS) spcos_hash_kernel(const HashParams P) {
    extern __shared__ __align__(16) unsigned char dyn[];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const unsigned lt = (1u << lane) - 1u;
    const int T = P.tile, K = P.k, n_tiles = P.n_tiles;
    unsigned char *base = dyn;
    unsigned *keys = reinterpret_cast<unsigned *>(base);                base += (size_t)H * 4;
    unsigned *vals = reinterpret_cast<unsigned *>(base);                base += (size_t)H * 4;
    HItem *items = reinterpret_cast<HItem *>(base);                     base += (size_t)HASH_ITEM_CAP * 16;
    uint2 *terms = reinterpret_cast<uint2 *>(base);                     base += (size_t)HASH_TERM_CAP * 8;    // {term, v_i}
    double *cq_score = reinterpret_cast<double *>(base);                base += (size_t)HASH_CQ * 8;
    int *cq_key = reinterpret_cast<int *>(base);                        base += (size_t)HASH_CQ * 4;
    int *wsum = reinterpret_cast<int *>(base);                          // [8] warp totals
    unsigned *wkth = reinterpret_cast<unsigned *>(base) + 8;            // [8] per-warp K-th lane maximum
    int *sh = reinterpret_cast<int *>(base) + 16;                       // [0] row, [1] queue length, [2] leftover flag, [3] ki
    unsigned *sh_thr = reinterpret_cast<unsigned *>(base) + 24;         // row threshold (fixed point)
    double *sh_kv = reinterpret_cast<double *>(base + 128);             // k-th key score

    for (int q = tid; q < H; q += HASH_NT) { keys[q] = HASH_EMPTY; vals[q] = 0u; }
    const int32_t *__restrict__ seg = P.seg;
    const int split = blockIdx.y;
    const int tiles_per = (P.n_tiles + P.n_splits - 1) / P.n_splits;
    const int tau_lo = split * tiles_per;
    const int tau_hi = min(P.n_tiles, tau_lo + tiles_per);
    int32_t *counter = P.counter + split;
    const unsigned thr0 = h_thr_q(fmax(P.min_sim, 0.0));
    __syncthreads();

    for (;;) {
        if (tid == 0) sh[0] = atomicAdd(counter, 1);
        __syncthreads();
        const int i = sh[0];
        __syncthreads();
        if (i >= P.n_from) break;
        const int a0 = P.a_indptr[i];
        const int m = P.a_indptr[i + 1] - a0;
        const int64_t self_j = P.from_base + i - P.to_base;
        const int self_loc = (P.self_match && self_j >= 0 && self_j < (int64_t)P.n_to) ? (int)self_j : -1;
        // top-k list of the row: registers of warp 0 (lane r = rank r)
        double tv = P.min_sim; int ti = -1;
        // exclusive lower key for paging (candidates must rank strictly after it)
        double xv = 0.0; int xi = -1; bool has_x = false;
        if (P.excl_val) { xv = P.excl_val[i]; xi = P.excl_idx[i]; has_x = xi >= 0; }
        if (tid == 0) { sh[3] = -1; sh_thr[0] = thr0; sh_kv[0] = P.min_sim; }
        if (m > HASH_TERM_CAP) { if (tid == 0) atomicExch(P.err_flag, 3); }
        const int mm = min(m, HASH_TERM_CAP);
        // the row's terms, and the postings they will visit in this split (upper bound of the distinct to-rows touched)
        int u_loc = 0;
        for (int e = tid; e < mm; e += HASH_NT) {
            const int t = P.a_indices[a0 + e];
            const double x = floor(P.a_data[a0 + e] * 4294967296.0);
            terms[e] = make_uint2((unsigned)t, x >= 4294967295.0 ? 0xffffffffu : (unsigned)(unsigned long long)x);
            u_loc += seg[(int64_t)t * n_tiles + tau_hi] - seg[(int64_t)t * n_tiles + tau_lo];
        }
#pragma unroll
        for (int d = 16; d; d >>= 1) u_loc += __shfl_xor_sync(FULL, u_loc, d);
        if (lane == 0) wsum[w] = u_loc;
        __syncthreads();
        int U = 0;
#pragma unroll
        for (int q = 0; q < HASH_WARPS; ++q) U += wsum[q];
        __syncthreads();
        if (U == 0) {                                          // nothing in common with this shard
            if (w == 0 && lane < K) { const size_t o = ((size_t)split * P.n_from + i) * K + lane; P.top_idx[o] = -1; P.top_val[o] = 0.0; }
            continue;
        }
        const int ntau = tau_hi - tau_lo;
        int n_pass = min(ntau, (U + H / 2 - 1) / (H / 2));
        if (n_pass < 1) n_pass = 1;
        const int tau_per = (ntau + n_pass - 1) / n_pass;

        for (int ps = 0; ps < n_pass; ++ps) {
            const int ta = tau_lo + ps * tau_per, tb = min(tau_hi, ta + tau_per);
            if (ta >= tb) break;
            const int ntp = tb - ta;
            const int npairs = mm * ntp;
            // The pass covers the to-rows [r_lo, r_lo + r_w) of each of its tiles -- normally the whole tile.  When the table
            // fills (a row that visits far more postings in these tiles than the estimate), the table is cleared and the range
            // halved, so no input can overflow it.
            int r_lo = 0, r_w = T;
            while (r_lo < T) {
            const unsigned f_lo = (unsigned)r_lo, f_hi = (unsigned)min(T, r_lo + r_w);
            if (tid == 0) sh[4] = 0;
            // ---- accumulate: (term, tile) segments -> work items -> hash inserts ------------------------------------
            for (int pb = 0; pb < npairs; pb += HASH_NT) {
                const int p = pb + tid;
                int s = 0, len = 0; unsigned keybase = 0u, v = 0u;
                if (p < npairs) {
                    const int e = p / ntp, tau = ta + (p - e * ntp);
                    const uint2 tt = terms[e];
                    v = tt.y;
                    const int64_t c = (int64_t)tt.x * n_tiles + tau;
                    s = seg[c];
                    len = seg[c + 1] - s;
                    keybase = (unsigned)tau * (unsigned)T;
                }
                const int nch = (len + 31) >> 5;
                const int incl = warp_incl_scan(nch);
                if (lane == 31) wsum[w] = incl;
                __syncthreads();
                int woff = 0, total = 0;
#pragma unroll
                for (int q = 0; q < HASH_WARPS; ++q) { const int x = wsum[q]; if (q < w) woff += x; total += x; }
                if (total == 0) { __syncthreads(); continue; }
                const int first = woff + incl - nch;
                for (int start = 0; start < total; start += HASH_ITEM_CAP) {
                    for (int c = 0; c < nch; ++c) {
                        const int id = first + c - start;
                        if (id >= 0 && id < HASH_ITEM_CAP) { HItem it; it.off = s + 32 * c; it.cnt = len - 32 * c; it.keybase = keybase; it.v = v; items[id] = it; }
                    }
                    __syncthreads();
                    const int nb = min(HASH_ITEM_CAP, total - start);
                    for (int q = w; q < nb; q += HASH_WARPS) {
                        const HItem it = items[q];
                        if (lane < it.cnt) {
                            const uint2 pk = __ldg(P.post_pk + it.off + lane);
                            if (pk.x >= f_lo && pk.x < f_hi) {
                                const unsigned key = it.keybase + pk.x;             // to-row local to the shard
                                const unsigned add = __umulhi(it.v, pk.y) + 1u;
                                unsigned h = (key * 2654435761u) >> (32 - LOGH);
                                bool done = false;
                                for (int probe = 0; probe < (H < 512 ? H : 512); ++probe) {
                                    const unsigned old = atomicCAS(&keys[h], HASH_EMPTY, key);
                                    if (old == HASH_EMPTY || old == key) { atomicAdd(&vals[h], add); done = true; break; }
                                    h = (h + 1) & (H - 1);
                                }
                                if (!done) sh[4] = 1;                               // table (nearly) full: this range is redone in halves
                            }
                        }
                    }
                    __syncthreads();
                }
            }
            if (sh[4] != 0 && r_w > 1) {                   // (uniform: written before the barrier that ends the accumulate phase)
                __syncthreads();
                for (int q = tid; q < H; q += HASH_NT) { keys[q] = HASH_EMPTY; vals[q] = 0u; }
                r_w = (r_w + 1) >> 1;
                __syncthreads();
                continue;
            }
            // ---- select: scan the table, exact re-scoring of the sums above the threshold --------------------------------
            unsigned gate = sh_thr[0];
            if (sh[3] < 0 && !has_x) {                     // (paging excludes rows by exact key: no pre-selection then)
                // list not full: per warp, the K-th largest of its 32 lane maxima is a lower bound of the pass's K-th best sum
                unsigned mx = 0u;
                for (int q = tid; q < H; q += HASH_NT) {
                    const unsigned key = keys[q];
                    if (key != HASH_EMPTY && (int)key != self_loc) mx = max(mx, vals[q]);
                }
                const unsigned srt = h_sort_desc(mx, lane);
                const unsigned kth = __shfl_sync(FULL, srt, K - 1);
                if (lane == 0) wkth[w] = kth;
                __syncthreads();
                unsigned best = 0u;
#pragma unroll
                for (int q = 0; q < HASH_WARPS; ++q) best = max(best, wkth[q]);
                if (best > K2H_MARGIN_Q) gate = max(gate, best - K2H_MARGIN_Q);
            }
            for (int sweep = 0; ; ++sweep) {
                if (tid == 0) { sh[1] = 0; sh[2] = 0; }
                __syncthreads();
                for (int q0 = 0; q0 < H; q0 += HASH_NT) {
                    const int q = q0 + tid;
                    const unsigned key = keys[q];
                    bool take = false;
                    if (key != HASH_EMPTY) {
                        const unsigned v = vals[q];
                        take = v > gate && (int)key != self_loc;
                        if (!take) { keys[q] = HASH_EMPTY; vals[q] = 0u; }
                    }
                    const unsigned tm = __ballot_sync(FULL, take);
                    if (tm) {
                        int slot = 0;
                        if (lane == 0) slot = atomicAdd(&sh[1], __popc(tm));
                        slot = __shfl_sync(FULL, slot, 0) + __popc(tm & lt);
                        if (take) {
                            if (slot < HASH_CQ) { cq_key[slot] = (int)key; keys[q] = HASH_EMPTY; vals[q] = 0u; }
                            else sh[2] = 1;                                          // queue full: this slot waits for the next sweep
                        }
                    }
                }
                __syncthreads();
                const int nq = min(sh[1], HASH_CQ);
                const bool more = sh[2] != 0;
                for (int q = tid; q < nq; q += HASH_NT) {
                    const int jloc = cq_key[q];
                    const int b0 = P.b_indptr[jloc];
                    cq_score[q] = h_exact_dot(P.a_indices + a0, P.a_data + a0, m, P.b_indices + b0, P.b_data + b0, P.b_indptr[jloc + 1] - b0);
                }
                __syncthreads();
                if (w == 0) {
                    double kv = sh_kv[0]; int ki = sh[3];
                    for (int q0 = 0; q0 < nq; q0 += 32) {
                        const int q = q0 + lane;
                        double sc = 0.0; int j = -1; bool cnd = false;
                        if (q < nq) {
                            sc = cq_score[q]; j = (int)(P.to_base + cq_key[q]); cnd = h_key_before(sc, j, kv, ki);
                            if (has_x && !h_key_before(xv, xi, sc, j)) cnd = false;
                        }
                        unsigned cm = __ballot_sync(FULL, cnd);
                        while (cm) {
                            const int src = __ffs(cm) - 1;
                            const double cs = shfl_d(sc, src);
                            const int cj = __shfl_sync(FULL, j, src);
                            const bool stays = (lane < K) && h_key_before(tv, ti, cs, cj);
                            const int pos = __popc(__ballot_sync(FULL, stays));
                            const double uv = __shfl_up_sync(FULL, tv, 1);
                            const int ui = __shfl_up_sync(FULL, ti, 1);
                            if (lane > pos) { tv = uv; ti = ui; }
                            else if (lane == pos) { tv = cs; ti = cj; }
                            kv = shfl_d(tv, K - 1);
                            ki = __shfl_sync(FULL, ti, K - 1);
                            cnd = cnd && lane != src && h_key_before(sc, j, kv, ki);
                            cm = __ballot_sync(FULL, cnd);
                        }
                    }
                    if (lane == 0) { sh_kv[0] = kv; sh[3] = ki; if (ki >= 0) sh_thr[0] = h_thr_q(kv); }
                }
                __syncthreads();
                if (!more) break;
                gate = max(gate, sh_thr[0]);
            }
            r_lo += r_w;
            }
        }
        if (w == 0 && lane < K) {
            const size_t o = ((size_t)split * P.n_from + i) * K + lane;
            P.top_idx[o] = ti;
            P.top_val[o] = (ti >= 0) ? tv : 0.0;
        }
        __syncthreads();
    }
}

template <int H, int LOGH>
static int launch_hash(const HashParams &P, int sms, int smem_max, cudaStream_t st) {
    const size_t arena = (hash_arena_bytes<H>() + 15) & ~(size_t)15;
    PFZ_REQUIRE(arena <= (size_t)smem_max, "pfz_spcos_topk_hash: %d slots need %zu B shared memory > %d available", H, arena, smem_max);
    PFZ_CUDA_OK(cudaFuncSetAttribute(spcos_hash_kernel<H, LOGH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)arena));
    int occ = 0;
    PFZ_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, spcos_hash_kernel<H, LOGH>, HASH_NT, arena));
    if (occ < 1) occ = 1;
    int gx = sms * occ;
    if (gx > P.n_from) gx = P.n_from;
    if (P.n_splits > 1) { gx = (gx + P.n_splits - 1) / P.n_splits; if (gx < 1) gx = 1; }
    spcos_hash_kernel<H, LOGH><<<dim3(gx, P.n_splits), HASH_NT, arena, st>>>(P);
    PFZ_LAUNCH_OK();
    return 0;
}

}  // namespace pfz

using namespace pfz;

extern "C" {

int pfz_spcos_topk_hash(const int32_t *a_indptr, const int32_t *a_indices, const double *a_data, int32_t n_from, const int32_t *seg,
                        const void *post_pk, const int32_t *b_indptr, const int32_t *b_indices, const double *b_data, int32_t tile,
                        int32_t n_tiles, int32_t n_to, int32_t k, double min_similarity, int32_t self_match, int64_t from_index_base,
                        int64_t to_index_base, int32_t n_splits, int32_t table_slots, const double *excl_val, const int32_t *excl_idx,
                        int32_t *top_idx, double *top_val, int32_t *row_counter, int32_t *err_flag_dev, void *stream) {
    PFZ_REQUIRE(k >= 1 && k <= 32, "pfz_spcos_topk_hash: k=%d unsupported (1..32)", k);
    PFZ_REQUIRE(tile >= 64 && tile <= 65536, "pfz_spcos_topk_hash: tile %d out of range", tile);
    PFZ_REQUIRE(n_splits >= 1 && n_splits <= n_tiles, "pfz_spcos_topk_hash: n_splits %d out of range", n_splits);
    PFZ_REQUIRE(table_slots == 1024 || table_slots == 2048 || table_slots == 8192 || table_slots == 16384, "pfz_spcos_topk_hash: table_slots %d must be 1024, 2048, 8192 or 16384", table_slots);
    if (n_from <= 0) return 0;
    cudaStream_t st = as_stream(stream);
    int dev = 0, sms = 0, smem_max = 0;
    PFZ_CUDA_OK(cudaGetDevice(&dev));
    PFZ_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    PFZ_CUDA_OK(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    PFZ_CUDA_OK(cudaMemsetAsync(row_counter, 0, sizeof(int32_t) * (size_t)n_splits, st));
    HashParams P{a_indptr, a_indices, a_data, n_from, seg, reinterpret_cast<const uint2 *>(post_pk), b_indptr, b_indices, b_data, tile, n_tiles,
                 n_to, k, min_similarity, self_match, from_index_base, to_index_base, n_splits, excl_val, excl_idx, top_idx, top_val, row_counter,
                 err_flag_dev};
    if (table_slots == 1024) return launch_hash<1024, 10>(P, sms, smem_max, st);
    if (table_slots == 2048) return launch_hash<2048, 11>(P, sms, smem_max, st);
    if (table_slots == 8192) return launch_hash<8192, 13>(P, sms, smem_max, st);
    return launch_hash<16384, 14>(P, sms, smem_max, st);
}
}
