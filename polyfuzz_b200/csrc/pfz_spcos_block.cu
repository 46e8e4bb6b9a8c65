// pfz_spcos_block.cu -- K2, from-row-BLOCK variant (PFZ_K2_BLOCK): sparse cosine + fused per-row top-k where a CTA of
// BF warps scores a block of BF from-rows (4, 8 or 16) against a to-tile at a time, so that ONE load of a posting chunk
// serves every from-row of the block that contains the term.
//
// Replaces sparse_dot_topn.awesome_cossim_topn (call site polyfuzz/models/_utils.py:82) and the reference's Python
// post-processing (polyfuzz/models/_utils.py:84-91, 128-146), like the other K2 variants (pfz_spcos.cu); results are
// bit-identical to them (same exact fp64 re-scoring, same ranking key).
//
// Why: the per-row kernels are bound by instruction issue -- most of it fetching postings and per-(row, tile)
// bookkeeping.  On name-like
// data a few hundred n-grams carry > 90 % of the postings ("inc", "llc", "cor", ...), so from-rows share their heavy
// terms.  Here
//   * from-rows are CLUSTERED by their three heaviest terms (sort of a 64-bit key), so a block of consecutive rows
//     shares most heavy terms (company names: one posting load serves ~4 of 8 rows on average);
//   * a block table (per block: distinct terms, per term the list of (row-in-block, weight)) is built once per call;
//   * accumulators acc[BF][tile] are FIXED-POINT sums in shared memory, updated with red.shared.add.u32: a
//     fire-and-forget integer atomic (a ld/fma/st read-modify-write chain serialises on the latency of each update;
//     float and 64-bit shared-memory adds are CAS loops).  Integer adds are associative, so the warps of the CTA share
//     one accumulator tile and consume the unit's work items (<= 32 postings of one term each) in any order, with no
//     hazards and no ordering.  Default: two 16-bit accumulators per word (unit 2^-15, to-rows j and j + tile/2 share
//     word j) -- twice the tile in the same shared memory; 32-bit accumulators (unit 2^-26) remain selectable;
//   * the sums only FILTER (as in PFZ_K2_DENSE32): after the unit's updates each warp scans (and clears) the
//     accumulators of ITS from-row against the row's gate (the K-th largest sum seen so far - margin, or a
//     lane-maxima bound while fewer than K sums have been seen); cells above it are queued and, at the end of the block,
//     re-scored exactly -- fp64, ascending terms, products rounded before the add -- by merging the two CSR rows.
// Fixed point, 16-bit: v16 = max(1, floor(v * 2^16)), w15 = max(1, round(w * 2^15)), update = ceil(v16 * w15 / 2^16):
// -1.01 < update - v*w*2^15 < 2.01 units and >= 1 for every common term; margin 4 m + 2 units for a from-row of m <= 128
// terms (every half-word stays below 2^15 + 258 < 2^16: no carry into its neighbour).  32-bit: v_i = floor(v * 2^32),
// w_i = round(w * 2^26), update = mulhi(v_i, w_i) + 1: -0.51 < update - v*w*2^26 <= 1.5 units, margin 1e-5.
#include <stdlib.h>
#include "pfz_common.cuh"

namespace pfz {

constexpr double K2B_SCALE = 67108864.0;         // 2^26: fixed-point unit of the accumulators
constexpr unsigned K2B_MARGIN_Q = 672u;          // 32-bit mode filter margin 1e-5 in units of 2^-26: >= 2 x 194 units (two approximate sums are compared)
constexpr int RANK_CAP = 16383;                  // term ranks are capped to 14 bits in the clustering key

struct __align__(16) BlockDesc { int pos0; int nrows; int base; int nterms; };

// ---- preparation kernels -------------------------------------------------------------------------------------
// terms sorted by document frequency in the to-shard, heaviest first: key = (~df) << 32 | term
__global__ void blk_term_key_kernel(const int32_t *__restrict__ seg, int n_vocab, int n_tiles, uint64_t *__restrict__ keys, int64_t n_pad) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_pad; t += (int64_t)gridDim.x * blockDim.x) {
        uint64_t k = ~0ull;
        if (t < n_vocab) {
            const uint32_t df = (uint32_t)(seg[(t + 1) * n_tiles] - seg[t * n_tiles]);
            k = ((uint64_t)(0xffffffffu - df) << 32) | (uint32_t)t;
        }
        keys[t] = k;
    }
}
__global__ void blk_term_rank_kernel(const uint64_t *__restrict__ keys, int n_vocab, int32_t *__restrict__ rank) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_vocab; i += gridDim.x * blockDim.x)
        rank[(uint32_t)(keys[i] & 0xffffffffu)] = min(i, RANK_CAP);
}
// from-row clustering key: the ranks of the row's three heaviest terms, then the row id (22 bits)
__global__ void blk_row_key_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices, const int32_t *__restrict__ rank,
                                   int n_from, uint64_t *__restrict__ keys, int64_t n_pad) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_pad; r += (int64_t)gridDim.x * blockDim.x) {
        uint64_t k = ~0ull;
        if (r < n_from) {
            int r1 = RANK_CAP, r2 = RANK_CAP, r3 = RANK_CAP;
            for (int p = indptr[r]; p < indptr[r + 1]; ++p) {
                const int x = rank[indices[p]];
                if (x < r1) { r3 = r2; r2 = r1; r1 = x; }
                else if (x < r2) { r3 = r2; r2 = x; }
                else if (x < r3) r3 = x;
            }
            k = ((uint64_t)r1 << 50) | ((uint64_t)r2 << 36) | ((uint64_t)r3 << 22) | (uint64_t)r;
        }
        keys[r] = k;
    }
}
__global__ void blk_perm_kernel(const uint64_t *__restrict__ keys, const int32_t *__restrict__ indptr, int n_from, int32_t *__restrict__ perm,
                                int32_t *__restrict__ nnz_perm) {
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p <= n_from; p += gridDim.x * blockDim.x) {
        if (p == n_from) { nnz_perm[p] = 0; continue; }
        const int r = (int)(keys[p] & 0x3fffffull);
        perm[p] = r;
        nnz_perm[p] = indptr[r + 1] - indptr[r];
    }
}

// Block tables: one warp per group of BF consecutive clustered positions.  A group whose rows hold more than FV_CAP
// entries is emitted as two descriptors of BF/2 rows (BF/2 x 128 <= FV_CAP); descriptor slots 2g, 2g+1 (nrows = 0: unused).
// Per descriptor, at offset base = pos_ptr[first position]:
//   blk_terms[base + u]  = u-th distinct term (ascending)
//   blk_fvdesc[base + u] = (start << 5) | count of its (row, weight) entries in blk_fv[base + start ...], rows ascending
//   blk_fv[base + e]     = { row-in-block * row_stride_bytes, v_i = floor(weight * 2^32) }
template <int BF>
__global__ void __launch_bounds__(128) blk_table_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                                        const double *__restrict__ data, int n_from, const int32_t *__restrict__ perm,
                                                        const int32_t *__restrict__ pos_ptr, int row_stride_bytes, int32_t *__restrict__ blk_terms,
                                                        int32_t *__restrict__ blk_fvdesc, uint2 *__restrict__ blk_fv, BlockDesc *__restrict__ descs,
                                                        int n_groups, int32_t *__restrict__ err_flag) {
    constexpr int FV_CAP = BF * 64;
    constexpr int WPB = BF == 16 ? 2 : 4;
    __shared__ uint32_t s_key[WPB][FV_CAP];
    __shared__ uint32_t s_val[WPB][FV_CAP];
    const int lane = lane_id(), w = threadIdx.x >> 5;
    const unsigned lt = (1u << lane) - 1u;
    if (w >= WPB) return;
    uint32_t *keys = s_key[w]; uint32_t *vals = s_val[w];
    for (int g = blockIdx.x * WPB + w; g < n_groups; g += gridDim.x * WPB) {
        const int p0 = g * BF, p1 = min(n_from, p0 + BF);
        const int total = pos_ptr[p1] - pos_ptr[p0];
        const int nsub = total <= FV_CAP ? 1 : 2;
        for (int sub = 0; sub < 2; ++sub) {
            BlockDesc d; d.pos0 = 0; d.nrows = 0; d.base = 0; d.nterms = 0;
            if (sub < nsub) {
                const int q0 = nsub == 1 ? p0 : min(p1, p0 + sub * (BF / 2));
                const int q1 = nsub == 1 ? p1 : min(p1, q0 + BF / 2);
                const int base = pos_ptr[q0];
                const int cnt = pos_ptr[q1] - base;
                if (cnt > FV_CAP) { if (lane == 0) atomicExch(err_flag, 1); }          // a row with > 128 terms: caller's contract broken
                else if (q1 > q0) {
                    for (int f = 0; f < q1 - q0; ++f) {
                        const int row = perm[q0 + f];
                        const int a0 = indptr[row], m = indptr[row + 1] - a0, o = pos_ptr[q0 + f] - base;
                        for (int e = lane; e < m; e += 32) {
                            keys[o + e] = ((uint32_t)indices[a0 + e] << 4) | (uint32_t)f;
                            const double x = floor(data[a0 + e] * 4294967296.0);
                            vals[o + e] = x >= 4294967295.0 ? 0xffffffffu : (uint32_t)(unsigned long long)x;
                        }
                    }
                    int P = 1;
                    while (P < cnt) P <<= 1;
                    for (int e = cnt + lane; e < P; e += 32) { keys[e] = 0xffffffffu; vals[e] = 0u; }
                    __syncwarp();
                    for (int k = 2; k <= P; k <<= 1) {
                        for (int j = k >> 1; j > 0; j >>= 1) {
                            for (int t = lane; t < (P >> 1); t += 32) {
                                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                                const int ix = i | j;
                                const uint32_t a = keys[i], b = keys[ix];
                                const bool up = (i & k) == 0;
                                if ((a > b) == up) { keys[i] = b; keys[ix] = a; const uint32_t va = vals[i]; vals[i] = vals[ix]; vals[ix] = va; }
                            }
                            __syncwarp();
                        }
                    }
                    int nd = 0;
                    for (int e0 = 0; e0 < cnt; e0 += 32) {
                        const int e = e0 + lane;
                        bool head = false; uint32_t term = 0;
                        if (e < cnt) {
                            const uint32_t key = keys[e];
                            term = key >> 4;
                            head = (e == 0) || (keys[e - 1] >> 4) != term;
                            blk_fv[base + e] = make_uint2((key & 15u) * (uint32_t)row_stride_bytes, vals[e]);
                        }
                        const unsigned hm = __ballot_sync(FULL, head);
                        if (head) {
                            int len = 1;
                            while (e + len < cnt && (keys[e + len] >> 4) == term) ++len;
                            const int u = nd + __popc(hm & lt);
                            blk_terms[base + u] = (int32_t)term;
                            blk_fvdesc[base + u] = (e << 5) | len;
                        }
                        nd += __popc(hm);
                    }
                    d.pos0 = q0; d.nrows = q1 - q0; d.base = base; d.nterms = nd;
                    __syncwarp();
                }
            }
            if (lane == 0) descs[2 * g + sub] = d;
        }
    }
}

// {tile-local row, w_i = round(weight * 2^26)} per posting, in segment order
__global__ void blk_pack_kernel(const uint16_t *__restrict__ post_idx, const double *__restrict__ post_val, const int32_t *__restrict__ nnz_ptr,
                                uint2 *__restrict__ post_pk) {
    const int64_t n = *nnz_ptr;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        post_pk[i] = make_uint2((uint32_t)post_idx[i], (uint32_t)__double2ll_rn(post_val[i] * 67108864.0));
}

// 16-bit mode: the posting already carries what the update needs -- x = byte offset of the accumulator WORD of the to-row
// (to-rows j and j + tile/2 share word j) | byte selector << 16 (0x4432: lower half-word, 0x3244: upper), y = w15 =
// max(1, round(weight * 2^15))
__global__ void blk_pack15_kernel(const uint16_t *__restrict__ post_idx, const double *__restrict__ post_val, const int32_t *__restrict__ nnz_ptr,
                                  int half_tile, uint2 *__restrict__ post_pk) {
    const int64_t n = *nnz_ptr;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t j = post_idx[i];
        const bool hi = j >= (uint32_t)half_tile;
        const uint32_t w15 = (uint32_t)max(1ll, __double2ll_rn(post_val[i] * 32768.0));
        post_pk[i] = make_uint2(((hi ? j - (uint32_t)half_tile : j) << 2) | ((hi ? 0x3244u : 0x4432u) << 16), w15);
    }
}

// ---- main kernel -----------------------------------------------------------------------------------------------
struct BlockParams {
    const int32_t *a_indptr; const int32_t *a_indices; const double *a_data; int n_from;
    const int32_t *perm; const BlockDesc *descs; int n_desc;
    const int32_t *blk_terms; const int32_t *blk_fvdesc; const uint2 *blk_fv;
    const int32_t *seg; const uint2 *post_pk;
    const int32_t *b_indptr; const int32_t *b_indices; const double *b_data;
    int tile, n_tiles, n_to, k; double min_sim; int self_match; int64_t from_base, to_base; int n_splits;
    int32_t *top_idx; double *top_val; int32_t *counter;
    int32_t *glist; int32_t *gcnt; int gcap;
};

__device__ __forceinline__ unsigned sm_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void red_add_u32(unsigned a, unsigned v) {
    // no "memory" clobber: the table loads of the following updates may be hoisted above it; every other shared-memory access
    // of the kernel is separated from the updates by __syncthreads()
    asm volatile("red.shared.add.u32 [%0], %1;" :: "r"(a), "r"(v));
}
__device__ __forceinline__ bool blk_key_before(double sa, int ia, double sb, int ib) { return (sa > sb) || (sa == sb && ia < ib); }
// canonical score of (from-row a, to-row b): common terms in ascending order, product rounded, then added.  The to-row is
// staged 32 entries at a time with INDEPENDENT loads (one memory latency per chunk instead of one per merge step -- the merge
// itself chases pointers), then merged against the from-row.
__device__ __noinline__ double blk_exact_dot(const int32_t *__restrict__ ai, const double *__restrict__ av, int an,
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
// descending bitonic sort of one value per lane: lane r ends up with the r-th largest
__device__ __forceinline__ unsigned warp_sort_desc_u32(unsigned x, int lane) {
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

// ---- main kernel (version 3) -----------------------------------------------------------------------------------
// Laid out for instruction count and registers (a monolithic version spilled to local memory in both loops and needed
// 5 barriers per (block, tile) unit):
//   * everything rare -- queueing candidates, maintaining the K largest sums, exact re-scoring, the top-k list -- lives in
//     NOINLINE functions whose state is in shared memory (B3Row), so the two hot loops (work items, scan) keep a handful of
//     registers and nothing spills;
//   * work items are allocated with one shared-memory atomic per warp (no block-wide scan), the segment offsets of the next tile
//     are prefetched during the current one, and a unit needs 2 barriers: [table | A | items (red) | B | scan of the own row];
//     the scan of tile t overlaps the table phase of tile t+1 (barrier A of t+1 is the one that protects the accumulators);
//   * idle lanes of a partial chunk add into 32 dump words behind their row's cells (ptxas does not predicate ATOMS: a
//     predicated red costs a divergent branch; a dump cell costs one select per item);
//   * the item loop keeps B3_DEPTH posting chunks in flight per warp;
//   * 16-bit mode: update = ceil(v16 * w15 / 2^16) placed in its half-word by one byte permute (IMAD + PRMT), v16 =
//     max(1, floor(v * 2^16)), w15 = max(1, round(w * 2^15)) pre-packed with the word offset and the permute selector
//     (pfz_index_pack_q15): -1.01 < update - v*w*2^15 < 2.01 units per product, >= 1 for every common term; margin 4 m + 2.
#ifndef PFZ_B3_ICAP_PER_ROW
#define PFZ_B3_ICAP_PER_ROW 64
#endif
// Register bound: 16 warps per SM, i.e. 128 registers per thread (2 CTAs of 8 rows).  The default 4 096-row tile needs 88 KB of
// shared memory per 8-row CTA, which stops at 2 CTAs per SM anyway; a 64-register bound (32 warps) only made the kernel spill.
// On an H100 the 4 096-row tile at this bound takes about a fifth less time than the 2 048-row tile at 64 registers (DESIGN §4.1).
#ifndef PFZ_B3_MIN_CTAS
#define PFZ_B3_MIN_CTAS(BF) (16 / (BF))
#endif
constexpr int B3_ICAP_PER_ROW = PFZ_B3_ICAP_PER_ROW;              // staged work items per unit = 64 x block rows; larger units walk the term table directly
constexpr int B3_QCAP = 128;                     // candidates a from-row may queue before they are re-scored exactly
#ifndef PFZ_B3_DEPTH
#define PFZ_B3_DEPTH 3
#endif
constexpr int B3_DEPTH = PFZ_B3_DEPTH;                      // posting chunks in flight per warp

struct __align__(16) B3Item { int off; int cnt; unsigned fva; int nf; };
// what the rare paths need of the kernel parameters (one copy per CTA in shared memory)
struct __align__(16) B3Ctx {
    const int32_t *a_indptr; const int32_t *a_indices; const double *a_data;
    const int32_t *b_indptr; const int32_t *b_indices; const double *b_data;
    int64_t to_base; double scale; int K; int T; int TW; int gcap;
    int32_t *glist; int64_t grow0;               // deferred candidates: list of row r at glist + (grow0 + r) * gcap (grow0 = split * n_from)
};
// filter / top-k state of one from-row (= one warp)
struct __align__(16) B3Row {
    double tv[32]; int ti[32];                   // exact top-k list, lane r = rank r
    unsigned av[32];                             // the K largest fixed-point sums seen (lane r = r-th largest)
    int cand[B3_QCAP];                           // queued candidates (local to-row ids)
    int row, self_loc, ncand; unsigned thr, akth, MQ, gate; int gcount;        // gcount: candidates already moved to the row's global list
};

// Exact scoring + insertion of a list of candidates (local to-row ids) of one from-row into its top-k list (tv / ti, lane r = rank r),
// 32 candidates per round, newest first.  kv / ki: the K-th key on return.
__device__ __forceinline__ void blk_exact_rounds(const int32_t *__restrict__ a_indptr, const int32_t *__restrict__ a_indices, const double *__restrict__ a_data,
                                                 const int32_t *__restrict__ b_indptr, const int32_t *__restrict__ b_indices, const double *__restrict__ b_data,
                                                 int64_t to_base, int K, int row, int self_loc, const int *cand, int ncand, double &tv, int &ti, double &kv, int &ki) {
    const int lane = threadIdx.x & 31;
    const int a0 = a_indptr[row], m = a_indptr[row + 1] - a0;
    kv = shfl_d(tv, K - 1); ki = __shfl_sync(FULL, ti, K - 1);
    while (ncand > 0) {
        const int n_round = min(32, ncand), off = ncand - n_round;
        double sc = 0.0; int j = -1; bool cnd = false;
        if (lane < n_round) {
            const int jloc = cand[off + lane];
            const int b0 = b_indptr[jloc];
            sc = blk_exact_dot(a_indices + a0, a_data + a0, m, b_indices + b0, b_data + b0, b_indptr[jloc + 1] - b0);
            j = (int)(to_base + jloc);
            cnd = blk_key_before(sc, j, kv, ki) && jloc != self_loc;
        }
        unsigned cm = __ballot_sync(FULL, cnd);
        while (cm) {
            const int src = __ffs(cm) - 1;
            const double cs = shfl_d(sc, src);
            const int cj = __shfl_sync(FULL, j, src);
            const bool stays = (lane < K) && blk_key_before(tv, ti, cs, cj);
            const int pos = __popc(__ballot_sync(FULL, stays));
            const double uv = __shfl_up_sync(FULL, tv, 1);
            const int ui = __shfl_up_sync(FULL, ti, 1);
            if (lane > pos) { tv = uv; ti = ui; }
            else if (lane == pos) { tv = cs; ti = cj; }
            kv = shfl_d(tv, K - 1);
            ki = __shfl_sync(FULL, ti, K - 1);
            cnd = cnd && lane != src && blk_key_before(sc, j, kv, ki);
            cm = __ballot_sync(FULL, cnd);
        }
        ncand = off;
    }
}
// in-kernel exact re-scoring of a row's queue (only when its global candidate list is full); raises thr to the K-th exact key
__device__ __noinline__ void blk3_drain(const B3Ctx *cx, B3Row *rs) {
    const int lane = threadIdx.x & 31;
    double tv = rs->tv[lane]; int ti = rs->ti[lane];
    double kv; int ki;
    blk_exact_rounds(cx->a_indptr, cx->a_indices, cx->a_data, cx->b_indptr, cx->b_indices, cx->b_data, cx->to_base, cx->K, rs->row, rs->self_loc,
                     rs->cand, rs->ncand, tv, ti, kv, ki);
    rs->tv[lane] = tv; rs->ti[lane] = ti;
    if (lane == 0) {
        rs->ncand = 0;
        if (ki >= 0) {
            const double y = kv * cx->scale - (double)rs->MQ;
            const unsigned t = y <= 0.0 ? 0u : (unsigned)__double2ll_rd(y);
            if (t > rs->thr) rs->thr = t;
        }
    }
    __syncwarp();
}
// The queue of a row moves to its list in global memory: the exact re-scoring of the whole list is a kernel of its own
// (blk_exact_kernel: one warp per row, nothing else in its way) instead of 11 % of this kernel's warp time plus a barrier wait at
// the end of every block.  A full list falls back to re-scoring here.
__device__ __noinline__ void blk3_flush(const B3Ctx *cx, B3Row *rs) {
    const int lane = threadIdx.x & 31;
    const int ncand = rs->ncand, g = rs->gcount;
    if (g + ncand <= cx->gcap) {
        int32_t *dst = cx->glist + (size_t)(cx->grow0 + rs->row) * cx->gcap + g;
        for (int q = lane; q < ncand; q += 32) dst[q] = rs->cand[q];
        __syncwarp();
        if (lane == 0) { rs->gcount = g + ncand; rs->ncand = 0; }
        __syncwarp();
    } else blk3_drain(cx, rs);
}

// largest accumulator of a 16-byte group: plain maximum, or the maximum over the 16-bit halves
template <bool P16>
__device__ __forceinline__ unsigned blk3_wmax(const uint4 &v) {
    if (!P16) return max(max(v.x, v.y), max(v.z, v.w));
    const unsigned m2 = __vmaxu2(__vmaxu2(v.x, v.y), __vmaxu2(v.z, v.w));
    return max(m2 & 0xffffu, m2 >> 16);
}

__device__ __forceinline__ uint4 lds128(unsigned a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ void sts128_zero(unsigned a) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" :: "r"(a), "r"(0u));
}
// Fewer than K sums seen so far: the K-th largest of the 32 lane maxima of the row bounds the unit's K-th best sum from below.
// Returns the gate for this scan.  row_s: shared-memory address of the row's cells.
template <bool P16>
__device__ __noinline__ unsigned blk3_first_gate(const B3Ctx *cx, const B3Row *rs, unsigned row_s) {
    const int lane = threadIdx.x & 31;
    const int ng = cx->TW >> 2;
    unsigned mx = 0u;
    for (int c = lane; c < ng; c += 32) mx = max(mx, blk3_wmax<P16>(lds128(row_s + ((unsigned)c << 4))));
    const unsigned srt = warp_sort_desc_u32(mx, lane);
    const unsigned kth = __shfl_sync(FULL, srt, cx->K - 1);
    unsigned gate = rs->gate;
    const unsigned MQ = rs->MQ;
    if (kth > MQ) gate = max(gate, kth - MQ);
    return gate;
}

// Filter state of a row while candidates are taken: registers of blk3_scan_slow for the whole row scan
struct B3St { unsigned av, akth, gate, MQ; int ncand; };
__device__ __forceinline__ B3St blk3_load_state(const B3Row *rs, int lane, unsigned gate) {
    B3St st; st.av = rs->av[lane]; st.akth = rs->akth; st.gate = gate; st.MQ = rs->MQ; st.ncand = rs->ncand; return st;
}
__device__ __forceinline__ void blk3_store_state(B3Row *rs, const B3St &st, int lane) {
    rs->av[lane] = st.av;
    if (lane == 0) { rs->akth = st.akth; rs->ncand = st.ncand; rs->gate = st.gate; }
    __syncwarp();
}
// One 16-byte group of accumulators at shared address `a` whose first cell is to-row `cellbase` and which holds a cell above
// the gate: the first lanes of the warp read ONE cell each (a half-word in 16-bit mode), vote, queue the cells above the gate
// and keep the K largest sums; a full queue moves to the row's global list.
template <bool P16>
__device__ __forceinline__ void blk3_take_group(const B3Ctx *cx, B3Row *rs, B3St &st, unsigned a, int cellbase, int lane, int K, int TW) {
    constexpr int NC = P16 ? 8 : 4;                                 // cells per 16-byte group
    unsigned x = 0u;
    if (lane < NC) {
        if (P16) { unsigned short h; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(a + 2u * (unsigned)lane)); x = h; }
        else asm volatile("ld.shared.u32 %0, [%1];" : "=r"(x) : "r"(a + 4u * (unsigned)lane));
    }
    const bool take = x > st.gate;
    unsigned tm = __ballot_sync(FULL, take);
    if (tm == 0u) return;
    if (st.ncand + NC > B3_QCAP) {                               // queue full: move it to the row's global list
        if (lane == 0) rs->ncand = st.ncand;
        __syncwarp();
        blk3_flush(cx, rs);
        st.ncand = 0;
        st.gate = max(st.gate, rs->thr);
    }
    if (take) rs->cand[st.ncand + __popc(tm & ((1u << lane) - 1u))] = cellbase + (P16 ? (lane >> 1) + ((lane & 1) ? TW : 0) : lane);
    st.ncand += __popc(tm);
    while (tm) {
        const int s2 = __ffs(tm) - 1; tm &= tm - 1;
        const unsigned cx2 = __shfl_sync(FULL, x, s2);
        if (cx2 <= st.akth) continue;
        const int pos = __popc(__ballot_sync(FULL, (lane < K) && st.av >= cx2));
        const unsigned up = __shfl_up_sync(FULL, st.av, 1);
        if (lane > pos) st.av = up; else if (lane == pos) st.av = cx2;
        st.akth = __shfl_sync(FULL, st.av, K - 1);
    }
    if (st.akth > st.MQ) st.gate = max(st.gate, st.akth - st.MQ);
}

// one posting chunk applied to the from-rows that hold the term (nf is warp-uniform); idle lanes (pk = 0) add into their dump word.
// 16-bit mode: pk = {word byte offset | selector << 16, w15}, update = ceil(v16 * w15 / 2^16) in its half-word (IMAD + PRMT);
// 32-bit mode: pk = {tile-local row, w_i}, update = mulhi(v_i, w_i) + 1.  The (row, weight) list is read two entries at a time
// and an odd tail takes one red of its own: every red adds a real product (69 % of the (block, term) pairs of company names
// have one row, so a red of weight 0 for the odd tail was 16 % of all reds).
template <bool P16>
__device__ __forceinline__ unsigned blk3_update(unsigned v, unsigned wq, unsigned sel) {
    if (P16) return __byte_perm(v * wq + 0xffffu, 0u, sel);
    return __umulhi(v, wq) + 1u;
}
__device__ __forceinline__ uint2 lds64(unsigned a) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
    return v;
}
template <bool P16>
__device__ __forceinline__ void blk3_process(int lane, int cnt, unsigned fva, int nf, uint2 pk, unsigned acc_s, unsigned dump_s) {
    unsigned cell, sel = 0u;
    const unsigned wq = pk.y;
    if (P16) { cell = acc_s + (pk.x & 0xffffu); sel = pk.x >> 16; }
    else cell = acc_s + (pk.x << 2);
    if (lane >= cnt) cell = dump_s;
#pragma unroll 1
    for (; nf >= 2; nf -= 2, fva += 16u) {
        const uint2 e0 = lds64(fva), e1 = lds64(fva + 8u);
        red_add_u32(cell + e0.x, blk3_update<P16>(e0.y, wq, sel));
        red_add_u32(cell + e1.x, blk3_update<P16>(e1.y, wq, sel));
    }
    if (nf) {
        const uint2 e0 = lds64(fva);
        red_add_u32(cell + e0.x, blk3_update<P16>(e0.y, wq, sel));
    }
}

// The item phase of one unit as its own function (own register allocation): warp w walks items w, w + W, ... with the posting
// chunks of the next B3_DEPTH items in flight.  items_s: shared address of the item array.  A slot behind the last item holds an
// empty item (cnt = nf = 0).
template <int W, bool P16>
__device__ __noinline__ void blk3_item_loop(unsigned items_s, int total, const uint2 *__restrict__ pk_lane, unsigned acc_s, unsigned dump_s) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int qc[B3_DEPTH], qn[B3_DEPTH]; unsigned qa[B3_DEPTH]; uint2 qp[B3_DEPTH];
#pragma unroll
    for (int d = 0; d < B3_DEPTH; ++d) {
        const int i = w + d * W;
        qc[d] = 0; qn[d] = 0; qa[d] = 0u; qp[d] = make_uint2(0u, 0u);
        if (i < total) {
            const uint4 it = lds128(items_s + ((unsigned)i << 4));            // {off, cnt, fva, nf}
            qc[d] = (int)it.y; qn[d] = (int)it.w; qa[d] = it.z;
            if (lane < (int)it.y) qp[d] = __ldg(pk_lane + (int)it.x);
        }
    }
#pragma unroll 1
    for (int i0 = w; i0 < total; i0 += B3_DEPTH * W) {
#pragma unroll
        for (int d = 0; d < B3_DEPTH; ++d) {
            blk3_process<P16>(lane, qc[d], qa[d], qn[d], qp[d], acc_s, dump_s);
            const int ni = i0 + (d + B3_DEPTH) * W;
            qc[d] = 0; qn[d] = 0; qp[d] = make_uint2(0u, 0u);
            if (ni < total) {
                const uint4 it = lds128(items_s + ((unsigned)ni << 4));
                qc[d] = (int)it.y; qn[d] = (int)it.w; qa[d] = it.z;
                if (lane < (int)it.y) qp[d] = __ldg(pk_lane + (int)it.x);
            }
        }
    }
}

// Scan + clear of one row.  The hot loop is a LEAF function (a call inside a loop makes ptxas keep the loop state in local
// memory): it clears 16-byte groups (two per lane and step) until one holds a cell above the gate, which it leaves in place
// and reports; the caller (blk3_scan_slow) takes the candidates of that step and resumes.
template <bool P16>
__device__ __noinline__ int blk3_scan_until_hit(unsigned row_s, int c, int ng, unsigned gate) {
#pragma unroll 1
    for (; c < ng; c += 64) {
        const unsigned a = row_s + ((unsigned)c << 4);
        const bool two = c + 32 < ng;
        const uint4 v0 = lds128(a);
        uint4 v1 = make_uint4(0u, 0u, 0u, 0u);
        if (two) v1 = lds128(a + 512u);
        if (__any_sync(FULL, max(blk3_wmax<P16>(v0), blk3_wmax<P16>(v1)) > gate)) break;
        sts128_zero(a);
        if (two) sts128_zero(a + 512u);
    }
    return c;
}
// The rest of a row scan once a step holds a cell above the gate (or while fewer than K sums have been seen: first != 0).
template <bool P16>
__device__ __noinline__ void blk3_scan_row(const B3Ctx *cx, B3Row *rs, unsigned row_s, int cell0) {
    const int lane = threadIdx.x & 31;
    const int ng = cx->TW >> 2;                                    // 16-byte groups of the row (a multiple of 32)
    unsigned gate0 = rs->gate;
    if (rs->akth == 0u) gate0 = blk3_first_gate<P16>(cx, rs, row_s);
    int c = blk3_scan_until_hit<P16>(row_s, lane, ng, gate0);
    if (c >= ng) {                                                 // the common case: nothing above the gate in this tile
        if (gate0 != rs->gate) { if (lane == 0) rs->gate = gate0; __syncwarp(); }
        return;
    }
    const int K = cx->K, TW = cx->TW;
    B3St st = blk3_load_state(rs, lane, gate0);                    // the filter state stays in registers for the rest of the row
    while (c < ng) {
        // the step at c holds a cell above the gate (two 16-byte groups per lane: c and c + 32)
        const unsigned a = row_s + ((unsigned)c << 4);
        const bool two = c + 32 < ng;
        const uint4 v0 = lds128(a);
        uint4 v1 = make_uint4(0u, 0u, 0u, 0u);
        if (two) v1 = lds128(a + 512u);
        const unsigned hl0 = __ballot_sync(FULL, blk3_wmax<P16>(v0) > st.gate), hl1 = __ballot_sync(FULL, blk3_wmax<P16>(v1) > st.gate);
        const int c_base = c - lane;
#pragma unroll 1
        for (int g = 0; g < 2; ++g) {
            unsigned hl = g == 0 ? hl0 : hl1;
#pragma unroll 1
            while (hl) {
                const int src = __ffs(hl) - 1; hl &= hl - 1;
                const int grp = c_base + src + 32 * g;
                blk3_take_group<P16>(cx, rs, st, row_s + ((unsigned)grp << 4), cell0 + grp * 4, lane, K, TW);
            }
        }
        sts128_zero(a);
        if (two) sts128_zero(a + 512u);
        c = blk3_scan_until_hit<P16>(row_s, c + 64, ng, st.gate);
    }
    blk3_store_state(rs, st, lane);
}

template <int BF, bool P16>
__host__ __device__ inline size_t blk3_arena_bytes(int T) {
    return (size_t)BF * (T * (P16 ? 2 : 4) + 128)   // acc: per from-row the tile's cells + 32 dump words (idle lanes)
           + (size_t)BF * B3_ICAP_PER_ROW * 16 // items
           + (size_t)BF * 64 * 8              // fv: (row, weight) table of the block
           + (size_t)BF * sizeof(B3Row)        // per-row filter / top-k state
           + sizeof(B3Ctx) + 64;               // context, counters
}

#ifdef PFZ_B3_TIMING
// developer instrumentation (build with PFZ_NVCC_EXTRA=-DPFZ_B3_TIMING, read with tools/b3_timing.py): SM cycles per phase,
// summed over the warps -- table, wait A, items, wait B, scan, exact re-scoring, wait at the end of the block
__device__ unsigned long long g_b3_cycles[8];
#define B3_TICK(slot)                                                                                \
    do { const long long _now = clock64(); if (lane == 0) atomicAdd(&g_b3_cycles[slot], (unsigned long long)(_now - _t)); _t = clock64(); } while (0)
#else
#define B3_TICK(slot) do { } while (0)
#endif

template <int BF, bool P16>
__global__ void __launch_bounds__(BF * 32, PFZ_B3_MIN_CTAS(BF)) spcos_blk3_kernel(const BlockParams P) {
    constexpr int W = BF, NT = BF * 32, FV_CAP = BF * 64, B3_ICAP = BF * B3_ICAP_PER_ROW;
    extern __shared__ __align__(16) unsigned char dyn[];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int T = P.tile;
    const int TW = P16 ? (T >> 1) : T;                                 // 32-bit accumulator words per from-row
    const int RW = TW + 32;                                            // row stride in words: cells + 32 dump words
    unsigned *acc = reinterpret_cast<unsigned *>(dyn);
    B3Item *items = reinterpret_cast<B3Item *>(dyn + (size_t)BF * RW * 4);
    uint2 *fvtab = reinterpret_cast<uint2 *>(reinterpret_cast<unsigned char *>(items) + (size_t)B3_ICAP * 16);
    B3Row *rs = reinterpret_cast<B3Row *>(reinterpret_cast<unsigned char *>(fvtab) + (size_t)FV_CAP * 8) + w;
    B3Ctx *cx = reinterpret_cast<B3Ctx *>(reinterpret_cast<unsigned char *>(fvtab) + (size_t)FV_CAP * 8 + (size_t)BF * sizeof(B3Row));
    int *misc = reinterpret_cast<int *>(cx + 1);
    int *icnt = misc;                                                   // [2] item counters (tile parity)
    int *bcast = misc + 2;
    int *wsum = misc + 4;                                               // [W <= 12]

    for (int q = tid; q < BF * RW; q += NT) acc[q] = 0u;
    if (tid < 4) misc[tid] = 0;
    if (tid == 0) {
        cx->a_indptr = P.a_indptr; cx->a_indices = P.a_indices; cx->a_data = P.a_data;
        cx->b_indptr = P.b_indptr; cx->b_indices = P.b_indices; cx->b_data = P.b_data;
        cx->to_base = P.to_base; cx->scale = P16 ? 32768.0 : K2B_SCALE; cx->K = P.k; cx->T = T; cx->TW = TW; cx->gcap = P.gcap;
        cx->glist = P.glist; cx->grow0 = (int64_t)blockIdx.y * P.n_from;
    }
    const unsigned acc_s = sm_u32(acc);
    const unsigned dump_s = acc_s + ((unsigned)(TW + lane) << 2);       // this lane's dump word of row 0
    const unsigned fv_s = sm_u32(fvtab);
    const unsigned items_s = sm_u32(items);
    const uint2 *pk_lane = P.post_pk + lane;
    const int32_t *__restrict__ seg = P.seg;
    const int n_tiles = P.n_tiles;
    const int split = blockIdx.y;
    const int tiles_per = (P.n_tiles + P.n_splits - 1) / P.n_splits;
    const int tau_lo = split * tiles_per;
    const int tau_hi = min(P.n_tiles, tau_lo + tiles_per);
    int32_t *counter = P.counter + split;
    __syncthreads();

    for (;;) {
        if (tid == 0) { bcast[0] = atomicAdd(counter, 1); icnt[0] = 0; icnt[1] = 0; }
        __syncthreads();
        const int di = bcast[0];
        __syncthreads();
        if (di >= P.n_desc) break;
        const BlockDesc D = P.descs[di];
        const int nrows = D.nrows, nterms = D.nterms;
        if (nrows == 0) continue;
        // warp w owns from-row w of the block
        const bool has_row = w < nrows;
        int stau = -1;
        {
            int row = 0, m = 0, sjl = 0;
            if (has_row) {
                row = P.perm[D.pos0 + w];
                m = P.a_indptr[row + 1] - P.a_indptr[row];
                const int64_t self_j = P.from_base + row - P.to_base;       // local to-row of the diagonal
                if (P.self_match && self_j >= 0 && self_j < (int64_t)P.n_to) { stau = (int)(self_j / T); sjl = (int)(self_j - (int64_t)stau * T); }
            }
            rs->tv[lane] = P.min_sim; rs->ti[lane] = -1; rs->av[lane] = 0u;
            if (lane == 0) {
                const unsigned MQ = P16 ? (unsigned)(4 * m + 2) : K2B_MARGIN_Q;  // filter margin in accumulator units (16-bit: -1.01 < update - exact < 2.01)
                const double y = fmax(P.min_sim, 0.0) * (P16 ? 32768.0 : K2B_SCALE) - (double)MQ;
                const unsigned thr = y <= 0.0 ? 0u : (unsigned)__double2ll_rd(y);
                rs->row = row; rs->self_loc = stau >= 0 ? stau * T + sjl : -1; rs->ncand = 0; rs->gcount = 0;
                rs->thr = thr; rs->akth = 0u; rs->MQ = MQ; rs->gate = thr;
                wsum[w] = m;
            }
        }
        // this thread's term (terms are dealt round-robin to the warps; first NT terms of the block, a block rarely has more):
        // segment row and (row, weight) list
        const int u_my = lane * W + w;
        int my_seg = 0; unsigned my_fva = 0u; int my_nf = 0;
        int pf_s = 0, pf_e = 0;
        if (u_my < nterms) {
            my_seg = P.blk_terms[D.base + u_my] * n_tiles;
            const unsigned fvd = (unsigned)P.blk_fvdesc[D.base + u_my];
            my_fva = fv_s + ((fvd >> 5) << 3); my_nf = (int)(fvd & 31u);
            pf_s = seg[my_seg + tau_lo]; pf_e = seg[my_seg + tau_lo + 1];
        }
        __syncthreads();
        {
            int nfv_total = 0;
#pragma unroll
            for (int q = 0; q < W; ++q) nfv_total += wsum[q];
            for (int e = tid; e < nfv_total; e += NT) {
                uint2 x = P.blk_fv[D.base + e];
                if (P16) x.y = max(1u, x.y >> 16);                      // v16 = max(1, floor(v * 2^16))
                fvtab[e] = x;
            }
        }
        // (the first barrier A below publishes fvtab and the row states)

#ifdef PFZ_B3_TIMING
        long long _t = clock64();
#endif
        for (int tau = tau_lo; tau < tau_hi; ++tau) {
            const int par = tau & 1;
            B3_TICK(4);                                                   // (scan of the previous tile / block prologue)
            // ---- table phase: one work item per 32 postings of a (term, tile) segment ----
            auto emit = [&](int s, int len, unsigned fva, int nf) {
                const int nch = (len + 31) >> 5;
                int first = 0;
                if (nch > 0) first = atomicAdd(&icnt[par], nch);         // (a handful of lanes per warp hold a term: cheaper than a warp scan)
                if (nch > 0 && first < B3_ICAP) { B3Item it; it.off = s; it.cnt = len; it.fva = fva; it.nf = nf; items[first] = it; }
                unsigned big = __ballot_sync(FULL, nch > 1);
                while (big) {                                             // the further chunks of long segments: written by the whole warp
                    const int src = __ffs(big) - 1; big &= big - 1;
                    const int s2 = __shfl_sync(FULL, s, src), l2 = __shfl_sync(FULL, len, src), f2 = __shfl_sync(FULL, first, src);
                    const unsigned a2 = __shfl_sync(FULL, fva, src); const int n2 = __shfl_sync(FULL, nf, src);
                    for (int c = 1 + lane; c < ((l2 + 31) >> 5); c += 32)
                        if (f2 + c < B3_ICAP) { B3Item it; it.off = s2 + 32 * c; it.cnt = l2 - 32 * c; it.fva = a2; it.nf = n2; items[f2 + c] = it; }
                }
            };
            if (w < nterms) {                                             // (warp-uniform: lane 0 holds term w)
                const int s = pf_s, len = pf_e - pf_s;
                if (u_my < nterms && tau + 1 < tau_hi) { pf_s = seg[my_seg + tau + 1]; pf_e = seg[my_seg + tau + 2]; }
                emit(s, u_my < nterms ? len : 0, my_fva, my_nf);
            }
            for (int tb = NT; tb < nterms; tb += NT) {                    // blocks with more than NT distinct terms (rare)
                if (tb + (w << 5) < nterms) {
                    const int u = tb + tid;
                    int s = 0, len = 0; unsigned fva = 0u; int nf = 0;
                    if (u < nterms) {
                        const int sb = P.blk_terms[D.base + u] * n_tiles + tau;
                        const unsigned fvd = (unsigned)P.blk_fvdesc[D.base + u];
                        s = seg[sb]; len = seg[sb + 1] - s; fva = fv_s + ((fvd >> 5) << 3); nf = (int)(fvd & 31u);
                    }
                    emit(s, len, fva, nf);
                }
            }
            B3_TICK(0);                                                   // table
            __syncthreads();                                              // ---- barrier A: items visible; every row of the previous tile scanned
            B3_TICK(1);                                                   // wait at A
            const int total = icnt[par];
            if (tid == 0) icnt[par ^ 1] = 0;
            if (total == 0) { __syncthreads(); continue; }                 // (uniform; the barrier orders the counter reset)

            if (total <= B3_ICAP) {
                blk3_item_loop<W, P16>(items_s, total, pk_lane, acc_s, dump_s);
            } else {
                // oversized unit: warps walk the term table directly (terms w, w + W, ...), chunk by chunk
                for (int u = w; u < nterms; u += W) {
                    const int sb = P.blk_terms[D.base + u] * n_tiles + tau;
                    const unsigned fvd = (unsigned)P.blk_fvdesc[D.base + u];
                    const int s = seg[sb], len = seg[sb + 1] - s;
                    for (int c = 0; c < len; c += 32) {
                        uint2 pk = make_uint2(0u, 0u);
                        if (lane < len - c) pk = __ldg(pk_lane + s + c);
                        blk3_process<P16>(lane, len - c, fv_s + ((fvd >> 5) << 3), (int)(fvd & 31u), pk, acc_s, dump_s);
                    }
                }
            }
            B3_TICK(2);                                                   // items
            __syncthreads();                                              // ---- barrier B: every update of the unit done
            B3_TICK(3);                                                   // wait at B
            // ---- scan + clear: warp w scans the accumulators of its row against the row's threshold ----
            if (has_row) {
                if (stau == tau) {                                     // the diagonal never competes
                    if (lane == 0) {
                        const int sjl = rs->self_loc - stau * T;
                        if (P16) acc[(size_t)w * RW + (sjl >= TW ? sjl - TW : sjl)] &= (sjl >= TW ? 0x0000ffffu : 0xffff0000u);
                        else acc[(size_t)w * RW + sjl] = 0u;
                    }
                    __syncwarp();
                }
                blk3_scan_row<P16>(cx, rs, acc_s + (unsigned)(w * RW) * 4u, tau * T);
            }
        }
        B3_TICK(4);
        if (has_row) {
            __syncwarp();
            blk3_flush(cx, rs);
            const size_t ro = (size_t)split * P.n_from + rs->row;
            if (lane < P.k) {                                          // the list as far as it was scored here (normally empty)
                const int ti = rs->ti[lane];
                P.top_idx[ro * P.k + lane] = ti;
                P.top_val[ro * P.k + lane] = (ti >= 0) ? rs->tv[lane] : 0.0;
            }
            if (lane == 0) P.gcnt[ro] = rs->gcount;
        }
        B3_TICK(5);                                                       // exact re-scoring at the end of the block
        __syncthreads();
        B3_TICK(6);                                                       // wait at the end of the block
    }
}

// Exact re-scoring of every row's candidate list (deferred from the main kernel): one warp per (split, from-row).
struct ExactParams {
    const int32_t *a_indptr; const int32_t *a_indices; const double *a_data;
    const int32_t *b_indptr; const int32_t *b_indices; const double *b_data;
    const int32_t *glist; const int32_t *gcnt; int gcap; int n_from; int n_splits; int n_to; int k; double min_sim; int self_match;
    int64_t from_base, to_base; int32_t *top_idx; double *top_val;
};
constexpr int EX_ROW_CAP = 128;                  // from-row terms staged in shared memory (the block kernel's contract; longer rows take the generic merge)
constexpr int EX_HASH = 2 * EX_ROW_CAP;          // open-addressed table of the staged from-row: load factor <= 1/2
__device__ __forceinline__ unsigned ex_slot(int t) { return ((unsigned)t * 0x9E3779B1u) >> 24; }   // (EX_HASH = 256 slots)
constexpr int EX_CHUNK = 8;                      // to-row entries loaded per step (independent loads)
__global__ void __launch_bounds__(256) blk_exact_kernel(const ExactParams P) {
    // The from-row is staged once per warp in a shared-memory hash table (term -> weight, linear probing); every lane scores one
    // candidate: it walks ITS to-row (entries loaded EX_CHUNK at a time, independent loads) and looks each term up in the table --
    // about 1.5 probes on average, where a binary search over the row took ceil(log2(m + 1)) dependent shared-memory loads.
    // Common terms are met in ascending order (the to-row's) and the products are rounded before the add: the canonical fp64
    // score, bit for bit.
    static_assert(EX_HASH == 256, "ex_slot() yields 8 bits");
    __shared__ int s_hk[8][EX_HASH];
    __shared__ double s_hv[8][EX_HASH];
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    const int64_t gw = (int64_t)blockIdx.x * 8 + wl;
    if (gw >= (int64_t)P.n_splits * P.n_from) return;
    const int n = P.gcnt[gw];
    if (n == 0) return;                                             // the main kernel's list (empty slots: -1, 0) stands
    const int row = (int)(gw % P.n_from), K = P.k;
    const int64_t self_j = P.from_base + row - P.to_base;
    const int self_loc = (P.self_match && self_j >= 0 && self_j < (int64_t)P.n_to) ? (int)self_j : -1;
    double tv = P.min_sim; int ti = -1;
    if (lane < K) { ti = P.top_idx[gw * K + lane]; if (ti >= 0) tv = P.top_val[gw * K + lane]; }
    double kv; int ki;
    const int a0 = P.a_indptr[row], m = P.a_indptr[row + 1] - a0;
    const int32_t *cand = P.glist + (size_t)gw * P.gcap;
    if (m > EX_ROW_CAP) {
        blk_exact_rounds(P.a_indptr, P.a_indices, P.a_data, P.b_indptr, P.b_indices, P.b_data, P.to_base, K, row, self_loc, cand, n, tv, ti, kv, ki);
    } else {
        int *hk = s_hk[wl]; double *hv = s_hv[wl];
        for (int s2 = lane; s2 < EX_HASH; s2 += 32) hk[s2] = -1;
        __syncwarp();
        for (int e = lane; e < m; e += 32) {                          // the row's terms are distinct: a slot is taken once
            const int t = P.a_indices[a0 + e];
            const double x = P.a_data[a0 + e];
            unsigned sl = ex_slot(t);
            while (atomicCAS(&hk[sl], -1, t) != -1) sl = (sl + 1) & (EX_HASH - 1);
            hv[sl] = x;
        }
        __syncwarp();
        kv = shfl_d(tv, K - 1); ki = __shfl_sync(FULL, ti, K - 1);
        int left = n;
        while (left > 0) {
            const int n_round = min(32, left), off = left - n_round;    // newest first
            double sc = 0.0; int j = -1; bool cnd = false;
            if (lane < n_round) {
                const int jloc = cand[off + lane];
                const int b0 = P.b_indptr[jloc], b1 = P.b_indptr[jloc + 1];
                for (int q = b0; q < b1; q += EX_CHUNK) {
                    int t[EX_CHUNK]; double wgt[EX_CHUNK];
#pragma unroll
                    for (int u = 0; u < EX_CHUNK; ++u) { t[u] = -1; wgt[u] = 0.0; if (q + u < b1) { t[u] = P.b_indices[q + u]; wgt[u] = P.b_data[q + u]; } }
#pragma unroll
                    for (int u = 0; u < EX_CHUNK; ++u) {
                        if (t[u] < 0) break;                                // (past the end of the to-row)
                        unsigned sl = ex_slot(t[u]);
                        int k;
                        while ((k = hk[sl]) != t[u] && k != -1) sl = (sl + 1) & (EX_HASH - 1);
                        if (k == t[u]) sc = __dadd_rn(sc, __dmul_rn(hv[sl], wgt[u]));
                    }
                }
                j = (int)(P.to_base + jloc);
                cnd = blk_key_before(sc, j, kv, ki) && jloc != self_loc;
            }
            unsigned cm = __ballot_sync(FULL, cnd);
            while (cm) {
                const int src = __ffs(cm) - 1;
                const double cs = shfl_d(sc, src);
                const int cj = __shfl_sync(FULL, j, src);
                const bool stays = (lane < K) && blk_key_before(tv, ti, cs, cj);
                const int pos = __popc(__ballot_sync(FULL, stays));
                const double uv = __shfl_up_sync(FULL, tv, 1);
                const int ui = __shfl_up_sync(FULL, ti, 1);
                if (lane > pos) { tv = uv; ti = ui; }
                else if (lane == pos) { tv = cs; ti = cj; }
                kv = shfl_d(tv, K - 1);
                ki = __shfl_sync(FULL, ti, K - 1);
                cnd = cnd && lane != src && blk_key_before(sc, j, kv, ki);
                cm = __ballot_sync(FULL, cnd);
            }
            left = off;
        }
    }
    if (lane < K) { P.top_idx[gw * K + lane] = ti; P.top_val[gw * K + lane] = (ti >= 0) ? tv : 0.0; }
}

template <int BF, bool P16>
static int launch_blk3(const BlockParams &P, int n_groups, int sms, int smem_max, cudaStream_t st) {
    size_t arena = (blk3_arena_bytes<BF, P16>(P.tile) + 15) & ~(size_t)15;
    { const char *e = getenv("PFZ_BLOCK_PAD_SMEM"); if (e) arena += (size_t)atoi(e); }      // developer knob: occupancy experiments
    PFZ_REQUIRE(arena <= (size_t)smem_max, "pfz_spcos_topk_block: tile %d x %d rows needs %zu B shared memory > %d available", P.tile, BF, arena, smem_max);
    PFZ_CUDA_OK(cudaFuncSetAttribute(spcos_blk3_kernel<BF, P16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)arena));
    int occ = 0;
    PFZ_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, spcos_blk3_kernel<BF, P16>, BF * 32, arena));
    if (occ < 1) occ = 1;
    int gx = sms * occ;
    if (gx > 2 * n_groups) gx = 2 * n_groups;
    if (P.n_splits > 1) { gx = (gx + P.n_splits - 1) / P.n_splits; if (gx < 1) gx = 1; }
    spcos_blk3_kernel<BF, P16><<<dim3(gx, P.n_splits), BF * 32, arena, st>>>(P);
    PFZ_LAUNCH_OK();
    return 0;
}

static int blk_grid(int64_t work, int threads, int cap) {
    int64_t g = (work + threads - 1) / threads;
    if (g < 1) g = 1;
    if (g > cap) g = cap;
    return (int)g;
}
static int64_t pow2_at_least(int64_t n) { int64_t p = 2; while (p < n) p <<= 1; return p; }
static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

struct BlockWs {
    size_t term_keys, term_rank, row_keys, perm, pos_ptr, scan_ws, blk_terms, blk_fvdesc, blk_fv, descs, counters, gcnt, glist, total;
};
constexpr int B3_GCAP = 192;                     // deferred candidates per (split, from-row); beyond that the main kernel re-scores in place
static BlockWs block_ws_layout(int64_t n_from, int64_t nnz_cap, int64_t n_vocab, int n_splits) {
    BlockWs L; size_t o = 0;
    const int64_t vp = pow2_at_least(n_vocab), np = pow2_at_least(n_from);
    const int64_t n_groups = (n_from + 3) / 4;                      // enough for every block size
    L.term_keys = o; o += align256((size_t)vp * 8);
    L.term_rank = o; o += align256((size_t)(n_vocab + 1) * 4);
    L.row_keys = o; o += align256((size_t)np * 8);
    L.perm = o; o += align256((size_t)(n_from + 1) * 4);
    L.pos_ptr = o; o += align256((size_t)(n_from + 2) * 4);
    L.scan_ws = o; o += align256((size_t)pfz_scan_ws_bytes(n_from + 2));
    L.blk_terms = o; o += align256((size_t)(nnz_cap + 1) * 4);
    L.blk_fvdesc = o; o += align256((size_t)(nnz_cap + 1) * 4);
    L.blk_fv = o; o += align256((size_t)(nnz_cap + 1) * 8);
    L.descs = o; o += align256((size_t)(2 * n_groups + 1) * sizeof(BlockDesc));
    L.counters = o; o += align256((size_t)(n_splits + 1) * 4);
    L.gcnt = o; o += align256((size_t)n_splits * (size_t)n_from * 4);
    L.glist = o; o += align256((size_t)n_splits * (size_t)n_from * B3_GCAP * 4);
    L.total = o;
    return L;
}

}  // namespace pfz

using namespace pfz;

extern "C" {

int64_t pfz_spcos_block_ws_bytes(int32_t n_from, int64_t nnz_cap_from, int32_t n_vocab, int32_t n_splits) {
    return (int64_t)block_ws_layout(n_from, nnz_cap_from, n_vocab, n_splits).total;
}

int64_t pfz_spcos_block_gcnt_offset(int32_t n_from, int64_t nnz_cap_from, int32_t n_vocab, int32_t n_splits) {
    return (int64_t)block_ws_layout(n_from, nnz_cap_from, n_vocab, n_splits).gcnt;
}

int pfz_index_pack_q26(const uint16_t *post_idx, const double *post_val, const int32_t *nnz_dev, void *post_pk, void *stream) {
    blk_pack_kernel<<<SM_COUNT * 8, 256, 0, as_stream(stream)>>>(post_idx, post_val, nnz_dev, reinterpret_cast<uint2 *>(post_pk));
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_index_pack_q15(const uint16_t *post_idx, const double *post_val, const int32_t *nnz_dev, int32_t tile, void *post_pk, void *stream) {
    PFZ_REQUIRE(tile >= 256 && tile <= 8192 && (tile % 256) == 0, "pfz_index_pack_q15: tile %d must be a multiple of 256 in 256..8192", tile);
    blk_pack15_kernel<<<SM_COUNT * 8, 256, 0, as_stream(stream)>>>(post_idx, post_val, nnz_dev, tile / 2, reinterpret_cast<uint2 *>(post_pk));
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_spcos_topk_block(const int32_t *a_indptr, const int32_t *a_indices, const double *a_data, int32_t n_from, int64_t nnz_cap_from,
                         const int32_t *seg, const void *post_pk, const int32_t *b_indptr, const int32_t *b_indices, const double *b_data,
                         int32_t n_vocab, int32_t tile, int32_t n_tiles, int32_t n_to, int32_t k, double min_similarity, int32_t self_match,
                         int64_t from_index_base, int64_t to_index_base, int32_t n_splits, int32_t block_rows, int32_t acc_bits, int32_t *top_idx,
                         double *top_val, int32_t *err_flag_dev, void *ws, void *stream) {
    PFZ_REQUIRE(k >= 1 && k <= 32, "pfz_spcos_topk_block: k=%d unsupported (1..32)", k);
    PFZ_REQUIRE(tile >= 128 && tile <= 4096 && (tile % 128) == 0, "pfz_spcos_topk_block: tile %d must be a multiple of 128 in 128..4096", tile);
    PFZ_REQUIRE(block_rows == 4 || block_rows == 8 || block_rows == 16, "pfz_spcos_topk_block: block_rows %d must be 4, 8 or 16", block_rows);
    PFZ_REQUIRE(acc_bits == 32 || (acc_bits == 16 && tile % 256 == 0), "pfz_spcos_topk_block: acc_bits %d must be 32, or 16 with a tile that is a multiple of 256", acc_bits);
    PFZ_REQUIRE(n_splits >= 1 && n_splits <= n_tiles, "pfz_spcos_topk_block: n_splits %d out of range", n_splits);
    PFZ_REQUIRE(n_from < (1 << 22), "pfz_spcos_topk_block: n_from %d exceeds the 22-bit row id of the clustering key", n_from);
    PFZ_REQUIRE(n_vocab < (1 << 28), "pfz_spcos_topk_block: n_vocab too large");
    if (n_from <= 0) return 0;
    cudaStream_t st = as_stream(stream);
    int dev = 0, sms = 0, smem_max = 0;
    PFZ_CUDA_OK(cudaGetDevice(&dev));
    PFZ_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    PFZ_CUDA_OK(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const BlockWs L = block_ws_layout(n_from, nnz_cap_from, n_vocab, n_splits);
    char *w = reinterpret_cast<char *>(ws);
    uint64_t *term_keys = reinterpret_cast<uint64_t *>(w + L.term_keys);
    int32_t *term_rank = reinterpret_cast<int32_t *>(w + L.term_rank);
    uint64_t *row_keys = reinterpret_cast<uint64_t *>(w + L.row_keys);
    int32_t *perm = reinterpret_cast<int32_t *>(w + L.perm);
    int32_t *pos_ptr = reinterpret_cast<int32_t *>(w + L.pos_ptr);
    int32_t *blk_terms = reinterpret_cast<int32_t *>(w + L.blk_terms);
    int32_t *blk_fvdesc = reinterpret_cast<int32_t *>(w + L.blk_fvdesc);
    uint2 *blk_fv = reinterpret_cast<uint2 *>(w + L.blk_fv);
    BlockDesc *descs = reinterpret_cast<BlockDesc *>(w + L.descs);
    int32_t *counters = reinterpret_cast<int32_t *>(w + L.counters);
    const int64_t vp = pow2_at_least(n_vocab), np = pow2_at_least(n_from);
    const int n_groups = (n_from + block_rows - 1) / block_rows;

    blk_term_key_kernel<<<blk_grid(vp, 256, SM_COUNT * 8), 256, 0, st>>>(seg, n_vocab, n_tiles, term_keys, vp);
    PFZ_LAUNCH_OK();
    if (pfz_sort_u64(term_keys, vp, stream)) return 1;
    blk_term_rank_kernel<<<blk_grid(n_vocab, 256, SM_COUNT * 8), 256, 0, st>>>(term_keys, n_vocab, term_rank);
    PFZ_LAUNCH_OK();
    blk_row_key_kernel<<<blk_grid(np, 256, SM_COUNT * 16), 256, 0, st>>>(a_indptr, a_indices, term_rank, n_from, row_keys, np);
    PFZ_LAUNCH_OK();
    if (pfz_sort_u64(row_keys, np, stream)) return 1;
    blk_perm_kernel<<<blk_grid(n_from + 1, 256, SM_COUNT * 16), 256, 0, st>>>(row_keys, a_indptr, n_from, perm, pos_ptr);
    PFZ_LAUNCH_OK();
    if (scan_exclusive_i32(pos_ptr, pos_ptr, (int64_t)n_from + 1, w + L.scan_ws, st)) return 1;
    const int row_stride = tile * (acc_bits == 16 ? 2 : 4) + 128;  // 32 dump words behind every row's cells
    if (block_rows == 4)
        blk_table_kernel<4><<<blk_grid((int64_t)n_groups * 32, 128, SM_COUNT * 16), 128, 0, st>>>(a_indptr, a_indices, a_data, n_from, perm, pos_ptr, row_stride,
                                                                                             blk_terms, blk_fvdesc, blk_fv, descs, n_groups, err_flag_dev);
    else if (block_rows == 8)
        blk_table_kernel<8><<<blk_grid((int64_t)n_groups * 32, 128, SM_COUNT * 16), 128, 0, st>>>(a_indptr, a_indices, a_data, n_from, perm, pos_ptr, row_stride,
                                                                                             blk_terms, blk_fvdesc, blk_fv, descs, n_groups, err_flag_dev);
    else
        blk_table_kernel<16><<<blk_grid((int64_t)n_groups * 32, 64, SM_COUNT * 16), 128, 0, st>>>(a_indptr, a_indices, a_data, n_from, perm, pos_ptr, row_stride,
                                                                                              blk_terms, blk_fvdesc, blk_fv, descs, n_groups, err_flag_dev);
    PFZ_LAUNCH_OK();
    PFZ_CUDA_OK(cudaMemsetAsync(counters, 0, sizeof(int32_t) * (size_t)n_splits, st));
    BlockParams P{a_indptr, a_indices, a_data, n_from, perm, descs, 2 * n_groups, blk_terms, blk_fvdesc, blk_fv, seg,
                  reinterpret_cast<const uint2 *>(post_pk), b_indptr, b_indices, b_data, tile, n_tiles, n_to, k, min_similarity, self_match,
                  from_index_base, to_index_base, n_splits, top_idx, top_val, counters,
                  reinterpret_cast<int32_t *>(w + L.glist), reinterpret_cast<int32_t *>(w + L.gcnt), B3_GCAP};
    int rc;
    if (block_rows == 4) rc = acc_bits == 16 ? launch_blk3<4, true>(P, n_groups, sms, smem_max, st) : launch_blk3<4, false>(P, n_groups, sms, smem_max, st);
    else if (acc_bits == 16) rc = block_rows == 8 ? launch_blk3<8, true>(P, n_groups, sms, smem_max, st) : launch_blk3<16, true>(P, n_groups, sms, smem_max, st);
    else rc = block_rows == 8 ? launch_blk3<8, false>(P, n_groups, sms, smem_max, st) : launch_blk3<16, false>(P, n_groups, sms, smem_max, st);
    if (rc) return rc;
    // exact re-scoring of the candidate lists the main kernel left behind
    ExactParams E{a_indptr, a_indices, a_data, b_indptr, b_indices, b_data, P.glist, P.gcnt, B3_GCAP, n_from, n_splits, n_to, k, min_similarity,
                  self_match, from_index_base, to_index_base, top_idx, top_val};
    const int64_t n_warps = (int64_t)n_splits * n_from;
    blk_exact_kernel<<<(unsigned)((n_warps + 7) / 8), 256, 0, st>>>(E);
    PFZ_LAUNCH_OK();
    return 0;
}

#ifdef PFZ_B3_TIMING
int pfz_debug_b3_cycles(unsigned long long *out8, int32_t reset) {
    PFZ_CUDA_OK(cudaDeviceSynchronize());
    PFZ_CUDA_OK(cudaMemcpyFromSymbol(out8, g_b3_cycles, sizeof(unsigned long long) * 8));
    if (reset) { unsigned long long z[8] = {0}; PFZ_CUDA_OK(cudaMemcpyToSymbol(g_b3_cycles, z, sizeof(z))); }
    return 0;
}
#endif
}
