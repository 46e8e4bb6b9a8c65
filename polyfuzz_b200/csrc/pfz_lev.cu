// pfz_lev.cu -- K3: all-pairs edit distance (bit-parallel Myers/Hyyro Levenshtein and Hyyro LCS/Indel) and
// Jaro / Jaro-Winkler similarity over the |from| x |to| grid with a fused per-row arg-best.
//
// Replaces rapidfuzz's scorer loop as the reference calls it:
//     polyfuzz/models/_rapidfuzz.py:99-113  process.extractOne(q, to_list, score_cutoff, scorer=fuzz.ratio)
//     polyfuzz/models/_distance.py:89-102   [scorer(q, t) for t in to_list]; np.argmax
//
// Mapping: one warp = one from-string (the bit-vector "pattern", its match masks Peq in shared memory),
// one lane = one to-string (the "text") at a time.  To-strings are pre-sorted by length and stored in
// groups of 32, transposed and packed 4 symbols per 32-bit word, so the 32 lanes of a warp read one
// coalesced 128-byte line per 4 dynamic-programming columns and run nearly the same trip count.
// Symbols are bytes: the host maps the code points that occur in the from-strings to 1..255 and every
// other code point to 0 ("matches nothing") -- equality among text-only symbols never matters.
//
// Patterns of <= 32 symbols use 32-bit words (half the integer work), <= 64 one 64-bit word, longer ones
// NW 64-bit blocks with horizontal carries (Hyyro 2003).  Work is integer-ALU bound (SURVEY.md 8d).
//
// Shared by the kernels here: the row driver of pfz_common.cuh (split_groups, claim_row, build_peq, WarpArgBest / WarpTopK,
// launch_rows), LevColumn (the Levenshtein / OSA column step of lev_kernel and dl_kernel), for_each_text_symbol (the text
// loop), dispatch_words (n_words -> <W, NW>) and run_k3 (the body of the C entry points).
#include "pfz_common.cuh"
#include <math_constants.h>
#include <cmath>

namespace pfz {

// ---- to-list layout ---------------------------------------------------------------------------
// sorted position p (by length) belongs to group p/32, lane p%32.
//   grp_word_off[g] : first 32-bit word of group g in `packed`; group g holds ceil(maxlen_g/4) x 32 words
//   slen[p], sorig[p]: length and original index of sorted string p
__global__ void __launch_bounds__(256) lev_pack_kernel(const uint32_t *__restrict__ blob, const int64_t *__restrict__ offsets,
                                                       const int32_t *__restrict__ order, int n_to, const uint8_t *__restrict__ sym_table,
                                                       const int64_t *__restrict__ grp_word_off, uint32_t *__restrict__ packed,
                                                       int32_t *__restrict__ slen) {
    const int lane = lane_id();
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    const int n_grp = (n_to + 31) >> 5;
    for (int g = gw; g < n_grp; g += nw) {
        const int p = g * 32 + lane;
        int64_t beg = 0; int len = 0;
        if (p < n_to) { const int o = order[p]; beg = offsets[o]; len = (int)(offsets[o + 1] - beg); slen[p] = len; }
        int mx = len;
#pragma unroll
        for (int d = 16; d; d >>= 1) mx = max(mx, __shfl_xor_sync(FULL, mx, d));
        const int nwords = (mx + 3) >> 2;
        uint32_t *dst = packed + grp_word_off[g];
        for (int wi = 0; wi < nwords; ++wi) {
            uint32_t word = 0;
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                const int q = wi * 4 + b;
                if (q < len) {
                    const uint32_t c = blob[beg + q];
                    word |= (uint32_t)(c < 0x110000u ? sym_table[c] : 0) << (8 * b);
                }
            }
            dst[(size_t)wi * 32 + lane] = word;
        }
    }
}

struct LevParams {
    const uint32_t *from_blob; const int64_t *from_off; const int32_t *from_ids; int n_ids;     // patterns of this class
    const uint8_t *sym_table;
    const uint32_t *packed; const int64_t *grp_word_off; const int32_t *slen; const int32_t *sorig; int n_to;
    int metric; double cutoff; int exclude_self; int64_t self_shift;
    double ratio_min_ns;                // RATIO: its cutoff as one test ns >= ratio_min_ns (ratio_min_ns_of)
    int n_splits;                       // to-groups are split over blockIdx.y
    int32_t *part_idx; double *part_score; int32_t *part_dist;     // [n_splits][n_from]
    int32_t *matrix; int64_t matrix_ld;                           // optional full matrix [n_from][n_to]
    int n_from; int32_t *counter;
    int k;                              // top-k epilogue: list length; part_idx / part_score are [n_splits][n_from][k]
};

__device__ __forceinline__ double ratio_ns(int d, int la, int lb) {      // Indel.normalized_similarity
    const int m = la + lb;
    return m ? 1.0 - (double)d / (double)m : 1.0;
}

__device__ __forceinline__ double score_of(int metric, int d, int la, int lb) {
    if (metric == PFZ_METRIC_NORM_LEV) { const int m = max(la, lb); return m ? 1.0 - (double)d / (double)m : 1.0; }
    return -(double)d;                  // raw distances: best = smallest
}

// RATIO's cutoff c in rapidfuzz's two steps: fuzz.ratio keeps ns only if ns >= c / 100 and returns ns * 100, then extractOne
// keeps that score only if ns * 100 >= c.  The steps disagree whenever (ns * 100) / 100 != ns (ns = 17/25 is rejected at
// c = 68.0).  Rounding is monotone, so {ns : ns * 100 >= c} is {ns >= t} for the least double t in it, and the two steps are
// the one test ns >= max(c / 100, t), found here once per launch.
static double ratio_min_ns_of(double c) {
    const double q = c / 100.0;
    if (!std::isfinite(q)) return q;                       // -inf: every pair, +inf / NaN: none (as both steps)
    double t = q;
    while (!(t * 100.0 >= c)) t = std::nextafter(t, HUGE_VAL);
    while (std::nextafter(t, -HUGE_VAL) * 100.0 >= c) t = std::nextafter(t, -HUGE_VAL);
    return t > q ? t : q;
}

// the row's slot of part_*: its k best (TOPK) or its arg-best
template <bool TOPK>
__device__ __forceinline__ void store_row(const LevParams &P, int i, const WarpTopK &top, WarpArgBest<> &best) {
    if constexpr (TOPK) {
        const size_t o = ((size_t)blockIdx.y * P.n_from + i) * P.k;
        top.store(P.part_idx + o, P.part_score + o);
    } else {
        const size_t o = (size_t)blockIdx.y * P.n_from + i;
        best.store(P.part_idx + o, P.part_score + o, P.part_dist + o);
    }
}

template <typename W> struct WordOps;
template <> struct WordOps<uint32_t> { static constexpr int BITS = 32; static __device__ __forceinline__ int pop(uint32_t x) { return __popc(x); } };
template <> struct WordOps<uint64_t> { static constexpr int BITS = 64; static __device__ __forceinline__ int pop(uint64_t x) { return __popcll(x); } };

// Calls f(symbol) for the n symbols of the lane's to-string (packed column src, 4 symbols per word).  The trip count is the
// warp's longest string, so the loop is warp-uniform, and the next word is loaded one word ahead: the recurrences f runs are
// long dependent chains.
template <typename F>
__device__ __forceinline__ void for_each_text_symbol(const uint32_t *src, int n, F &&f) {
    int nmax = n;
#pragma unroll
    for (int d = 16; d; d >>= 1) nmax = max(nmax, __shfl_xor_sync(FULL, nmax, d));
    uint32_t nextw = nmax > 0 ? src[0] : 0u;
    for (int j0 = 0; j0 < nmax; j0 += 4) {
        const uint32_t word = nextw;
        if (j0 + 4 < nmax) nextw = src[(size_t)((j0 >> 2) + 1) * 32];
#pragma unroll
        for (int bb = 0; bb < 4; ++bb) {
            if (j0 + bb < n) f((int)((word >> (8 * bb)) & 0xff));
        }
    }
}

// One bit-parallel column of Levenshtein (Myers 1999, blocks: Hyyro 2003) or, with OSA, of optimal string alignment (Hyyro
// 2003's transposition extension: D0 and the match masks of the previous text symbol are kept per block, DESIGN.md 4.9).
// step() takes the text symbol's match masks peq[s * NW ..] and returns the horizontal delta of pattern row m.
template <typename W, int NW, bool OSA>
struct LevColumn {
    static constexpr int B = WordOps<W>::BITS;
    W Pv[NW], Mv[NW];
    W D0[NW], PMo[NW];                                    // OSA: D0 and Peq of the previous text symbol
    __device__ __forceinline__ void init() {
#pragma unroll
        for (int b = 0; b < NW; ++b) {
            Pv[b] = ~(W)0; Mv[b] = 0;
            if constexpr (OSA) { D0[b] = 0; PMo[b] = 0; }     // PMo = 0: no transposition at the first symbol
        }
    }
    __device__ __forceinline__ int step(const W *eq, int last_blk, int last_bit) {
        int hin = 1;                                      // D[0][j] - D[0][j-1] = +1
        W trc = 0;                                        // OSA: top bit of the block below's X
#pragma unroll
        for (int b = 0; b < NW; ++b) {
            if (b <= last_blk) {
                W Eq = eq[b];
                const W pv = Pv[b], mv = Mv[b];
                if constexpr (!OSA) {
                    const W Xv = Eq | mv;
                    if (hin < 0) Eq |= 1;
                    const W Xh = (((Eq & pv) + pv) ^ pv) | Eq;
                    W Ph = mv | ~(Xh | pv);
                    W Mh = pv & Xh;
                    const int top = (b == last_blk) ? last_bit : B - 1;
                    const int hout = (int)((Ph >> top) & 1) - (int)((Mh >> top) & 1);
                    Ph <<= 1; Mh <<= 1;
                    if (hin < 0) Mh |= 1; else if (hin > 0) Ph |= 1;
                    Pv[b] = Mh | ~(Xv | Ph);
                    Mv[b] = Ph & Xv;
                    hin = hout;
                } else {
                    // X: rows that match this symbol where the previous column had no diagonal zero;
                    // one row up and ANDed with the previous symbol's matches, it marks a swap of b[j-1], b[j]
                    const W X = ~D0[b] & Eq;
                    const W TR = ((X << 1) | trc) & PMo[b];
                    trc = X >> (B - 1);
                    PMo[b] = Eq;
                    if (hin < 0) Eq |= 1;
                    const W D0n = (((Eq & pv) + pv) ^ pv) | Eq | mv | TR;
                    W Ph = mv | ~(D0n | pv);
                    W Mh = D0n & pv;
                    const int top = (b == last_blk) ? last_bit : B - 1;
                    const int hout = (int)((Ph >> top) & 1) - (int)((Mh >> top) & 1);
                    Ph <<= 1; Mh <<= 1;
                    if (hin < 0) Mh |= 1; else if (hin > 0) Ph |= 1;
                    Pv[b] = Mh | ~(D0n | Ph);
                    Mv[b] = Ph & D0n;
                    D0[b] = D0n;
                    hin = hout;
                }
            }
        }
        return hin;
    }
};

// One warp scores pattern `pat` against every to-string of its split.  LCS = false: Levenshtein, or with OSA = true optimal
// string alignment (LevColumn); LCS = true: longest common subsequence (Hyyro 2004) -> Indel = la + lb - 2*LCS.
// TOPK = false: per-row arg-best; TOPK = true: the k best per row in a WarpTopK, offered after every group of 32 to-strings.
// (minimum 1 block per SM for TOPK: without it ptxas's register target makes some top-k classes spill; 0 = unspecified)
template <typename W, int NW, bool LCS, int WARPS, bool TOPK = false, bool OSA = false>
__global__ void __launch_bounds__(WARPS * 32, TOPK ? 1 : 0) lev_kernel(const LevParams P) {
    static_assert(!(OSA && LCS), "OSA extends the Levenshtein recurrence");
    constexpr int B = WordOps<W>::BITS;
    extern __shared__ __align__(16) unsigned char dyn[];
    const int lane = lane_id();
    const int w = threadIdx.x >> 5;
    W *peq = reinterpret_cast<W *>(dyn) + (size_t)w * 256 * NW;              // peq[sym * NW + block]

    for (;;) {
        const int i = claim_row(P.counter + blockIdx.y, P.from_ids, P.n_ids);
        if (i < 0) break;
        const GroupRange gr = split_groups(P.n_to, P.n_splits);    // per row: held across rows, ptxas spilled it (LCS, 8+ words)
        const int64_t fb = P.from_off[i];
        const int m = (int)(P.from_off[i + 1] - fb);
        build_peq<W, NW>(peq, P.from_blob + fb, m, P.sym_table);
        const int last_bit = (m - 1) & (B - 1);          // bit of row m inside the last block (m > 0)
        const int last_blk = m > 0 ? (m - 1) / B : 0;

        WarpArgBest<> best;
        WarpTopK top;
        if constexpr (TOPK) top.init(P.k); else best.init();
        for (int g = gr.lo; g < gr.hi; ++g) {
            double cand_s = 0.0; int cand_j = -1;
            const int p = g * 32 + lane;
            const bool have = p < P.n_to;
            const int n = have ? P.slen[p] : 0;
            const int orig = have ? P.sorig[p] : -1;
            const uint32_t *src = P.packed + P.grp_word_off[g] + lane;
            int dist;
            if constexpr (!LCS) {
                LevColumn<W, NW, OSA> col;
                col.init();
                int score = m;
                for_each_text_symbol(src, n, [&](int s) { score += col.step(peq + s * NW, last_blk, last_bit); });
                dist = m > 0 ? score : n;
            } else {
                W S[NW];
#pragma unroll
                for (int b = 0; b < NW; ++b) S[b] = ~(W)0;
                for_each_text_symbol(src, n, [&](int s) {
                    unsigned carry = 0;
#pragma unroll
                    for (int b = 0; b < NW; ++b) {
                        if (b <= last_blk) {
                            const W Eq = peq[s * NW + b];
                            const W x = S[b], u = x & Eq;
                            // S' = (S + (S & Eq)) | (S - (S & Eq)); u is a subset of x, so x - u = x & ~Eq (no borrow);
                            // the addition carries across blocks
                            const W sum = x + u; unsigned c1 = sum < x; const W sum2 = sum + carry; c1 |= (sum2 < sum); carry = c1;
                            S[b] = sum2 | (x & ~Eq);
                        }
                    }
                });
                int lcs = 0;
#pragma unroll
                for (int b = 0; b < NW; ++b) {
                    if (m > 0 && b <= last_blk) {
                        W z = ~S[b];
                        if (b == last_blk && last_bit != B - 1) z &= (((W)1 << (last_bit + 1)) - 1);
                        lcs += WordOps<W>::pop(z);
                    }
                }
                dist = m + n - 2 * lcs;
            }
            if (have) {
                if (P.matrix) P.matrix[(int64_t)i * P.matrix_ld + orig] = dist;
                bool ok = !(P.exclude_self && (int64_t)orig == (int64_t)i + P.self_shift);
                double sc;
                if constexpr (LCS) {                    // RATIO: ns * 100 with the two-step cutoff; INDEL: the distance
                    const bool ratio = P.metric == PFZ_METRIC_RATIO;
                    const double ns = ratio ? ratio_ns(dist, m, n) : 0.0;
                    sc = ratio ? ns * 100.0 : -(double)dist;
                    if (ratio && !(ns >= P.ratio_min_ns)) ok = false;
                } else {
                    // OSA scores like Levenshtein: NORM_OSA takes NORM_LEV's expression and cutoff, raw OSA is a distance
                    sc = OSA ? score_of(P.metric == PFZ_METRIC_NORM_OSA ? PFZ_METRIC_NORM_LEV : PFZ_METRIC_LEV, dist, m, n)
                             : score_of(P.metric, dist, m, n);
                    if ((OSA ? P.metric == PFZ_METRIC_NORM_OSA : P.metric == PFZ_METRIC_NORM_LEV) && !(sc >= P.cutoff)) ok = false;
                }
                if constexpr (TOPK) { cand_s = sc; cand_j = ok ? orig : -1; }
                else if (ok) best.offer(sc, orig, dist);
            }
            if constexpr (TOPK) top.offer(cand_s, cand_j);
        }
        store_row<TOPK>(P, i, top, best);
        __syncwarp();
    }
}

// Jaro / Jaro-Winkler (jellyfish's definition, s1 = pattern = from-string, s2 = text = to-string).  The text-driven greedy:
// text symbol j takes the LOWEST unflagged pattern position i with |i - j| <= R and P[i] == T[j]; it flags the same pairs
// as the definition's pattern-driven loop (rapidfuzz's bit-parallel Jaro).  Pflag holds the flagged pattern bits; the
// lane records its matched text symbols in order in shared memory (<= min(m, n) bytes, column `lane` of the warp's
// store), so the transposition count pairs the k-th stored symbol with the k-th lowest Pflag bit: a mismatch iff
// bit i of Peq[stored k] is clear.  Scores are the definition's float64 expression, rounded step by step.
template <typename W>
__device__ __forceinline__ W window_bits(int lo, int hi) {      // bits lo..hi of one block (block-relative, may lie outside)
    constexpr int B = WordOps<W>::BITS;
    if (hi < 0 || lo >= B) return 0;
    const W up = hi >= B - 1 ? ~(W)0 : (((W)1 << (hi + 1)) - 1);
    const W dn = lo <= 0 ? ~(W)0 : ~(((W)1 << lo) - 1);
    return up & dn;
}

template <typename W> __device__ __forceinline__ int low_bit(W x);
template <> __device__ __forceinline__ int low_bit<uint32_t>(uint32_t x) { return __ffs(x) - 1; }
template <> __device__ __forceinline__ int low_bit<uint64_t>(uint64_t x) { return __ffsll(x) - 1; }

template <typename W, int NW, int WARPS, bool TOPK = false>
__global__ void __launch_bounds__(WARPS * 32) jaro_kernel(const LevParams P) {
    constexpr int B = WordOps<W>::BITS;
    constexpr int STORE = B * NW;                                           // max matches per lane
    extern __shared__ __align__(16) unsigned char dyn[];
    const int lane = lane_id();
    const int w = threadIdx.x >> 5;
    W *peq = reinterpret_cast<W *>(dyn) + (size_t)w * 256 * NW;              // peq[sym * NW + block]
    uint8_t *store = dyn + (size_t)WARPS * 256 * NW * sizeof(W) + (size_t)w * STORE * 32 + lane;    // store[k * 32]
    const bool winkler = P.metric == PFZ_METRIC_JARO_WINKLER;
    const GroupRange gr = split_groups(P.n_to, P.n_splits);

    for (;;) {
        const int i = claim_row(P.counter + blockIdx.y, P.from_ids, P.n_ids);
        if (i < 0) break;
        const int64_t fb = P.from_off[i];
        const int m = (int)(P.from_off[i + 1] - fb);
        build_peq<W, NW>(peq, P.from_blob + fb, m, P.sym_table);
        const int last_blk = m > 0 ? (m - 1) / B : 0;                          // blocks above it hold no pattern bits

        WarpArgBest<> best;
        WarpTopK top;
        if constexpr (TOPK) top.init(P.k); else best.init();
        for (int g = gr.lo; g < gr.hi; ++g) {
            double cand_s = 0.0; int cand_j = -1;
            const int p = g * 32 + lane;
            const bool have = p < P.n_to;
            const int n = have ? P.slen[p] : 0;
            const int orig = have ? P.sorig[p] : -1;
            const int R = max(0, max(m, n) / 2 - 1);
            const int jend = m > 0 ? min(n, m + R) : 0;                  // text positions >= m + R have an empty window
            int jmax = jend;
#pragma unroll
            for (int d = 16; d; d >>= 1) jmax = max(jmax, __shfl_xor_sync(FULL, jmax, d));
            const uint32_t *src = P.packed + P.grp_word_off[g] + lane;
            const uint32_t first = n > 0 ? src[0] : 0u;
            W F[NW], win[NW];                                                // win: pattern bits j-R .. j+R
#pragma unroll
            for (int b = 0; b < NW; ++b) { F[b] = 0; win[b] = window_bits<W>(-b * B, R - b * B); }
            int k = 0;
            uint32_t nextw = first;
            for (int j0 = 0; j0 < jmax; j0 += 4) {
                const uint32_t word = nextw;
                if (j0 + 4 < jmax) nextw = src[(size_t)((j0 >> 2) + 1) * 32];
#pragma unroll
                for (int bb = 0; bb < 4; ++bb) {
                    const int j = j0 + bb;
                    const int s = (word >> (8 * bb)) & 0xff;
                    if (j < jend && s) {
                        bool found = false;
#pragma unroll
                        for (int b = 0; b < NW; ++b) {
                            if (b <= last_blk) {
                                const W x = peq[s * NW + b] & ~F[b] & win[b];
                                if (!found && x) { F[b] |= x & (~x + 1); found = true; }
                            }
                        }
                        if (found) { store[(size_t)k * 32] = (uint8_t)s; ++k; }
                    }
                    // slide the window one position: shift left across blocks; bit 0 stays set while j + 1 <= R
#pragma unroll
                    for (int b = NW - 1; b >= 0; --b) {
                        if (b <= last_blk) win[b] = (win[b] << 1) | (b > 0 ? win[b > 0 ? b - 1 : 0] >> (B - 1) : (W)(j + 1 <= R));
                    }
                }
            }
            int trans = 0, kk = 0;
#pragma unroll
            for (int b = 0; b < NW; ++b) {
                W f = F[b];
                while (f) {
                    const int bit = low_bit<W>(f);
                    f &= f - 1;
                    const int s = store[(size_t)kk * 32];
                    ++kk;
                    trans += !((peq[s * NW + b] >> bit) & 1);
                }
            }
            double sc = 0.0;
            if (k > 0) {
                const double dm = (double)k;
                sc = __ddiv_rn(__dadd_rn(__dadd_rn(__ddiv_rn(dm, (double)m), __ddiv_rn(dm, (double)n)), __ddiv_rn(__dsub_rn(dm, (double)(trans / 2)), dm)), 3.0);
                if (winkler && sc > 0.7) {
                    const int cap = min(min(m, n), 4);
                    int pre = 0;
                    while (pre < cap && ((peq[((first >> (8 * pre)) & 0xff) * NW] >> pre) & 1)) ++pre;
                    if (pre > 0) sc = __dadd_rn(sc, __dmul_rn(__dmul_rn((double)pre, 0.1), __dsub_rn(1.0, sc)));
                }
            }
            if (have) {
                bool ok = !(P.exclude_self && (int64_t)orig == (int64_t)i + P.self_shift) && sc >= P.cutoff;
                if constexpr (TOPK) { cand_s = sc; cand_j = ok ? orig : -1; }
                else if (ok) best.offer(sc, orig, k);
            }
            if constexpr (TOPK) top.offer(cand_s, cand_j);
        }
        store_row<TOPK>(P, i, top, best);
        __syncwarp();
    }
}

__global__ void lev_merge_kernel(const int32_t *__restrict__ part_idx, const double *__restrict__ part_score, const int32_t *__restrict__ part_dist,
                                 int n_splits, int n_from, int32_t *__restrict__ best_idx, double *__restrict__ best_score,
                                 int32_t *__restrict__ best_dist) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_from; i += gridDim.x * blockDim.x) {
        double bs = 0.0; int bj = -1, bd = -1;
        for (int s = 0; s < n_splits; ++s) {
            const size_t o = (size_t)s * n_from + i;
            const int j = part_idx[o];
            if (j < 0) continue;
            const double sc = part_score[o];
            if (bj < 0 || WarpTopK::before(sc, j, bs, bj)) { bs = sc; bj = j; bd = part_dist[o]; }
        }
        best_idx[i] = bj; best_score[i] = bj >= 0 ? bs : 0.0; best_dist[i] = bd;
    }
}

// ---- unrestricted Damerau-Levenshtein (DESIGN.md 4.10) ------------------------------------------------------------------
// Per pair the warp computes OSA bit-parallel (the recurrence of lev_kernel<..., OSA = true>), which brackets DL:
//     max(ceil(2*osa/3), |m - n|) <= dl <= osa.
// A pair whose score upper bound is below the row's gate (a proven lower bound of its k-th best score) or below the running
// k-th exact score is dropped; if the two bounds meet the score is exact; otherwise the pair is queued, and every 32 queued
// pairs (and at the end of the row) all lanes run the exact DP, one pair each.  Matrix mode runs the DP on every pair.
constexpr int DL_NONE = 32000;          // RK: no earlier text occurrence (larger than any real term: distances are <= j + m)

template <typename W, int NW>
struct DlLayout {                       // one warp's shared memory
    static constexpr int MAXM = WordOps<W>::BITS * NW;
    static constexpr size_t PEQ = (size_t)256 * NW * sizeof(W);
    static constexpr size_t QUEUE = 32 * sizeof(int2);                                  // (sorted to-position, lower bound)
    static constexpr size_t STATE = (size_t)3 * (MAXM + 1) * 32 * sizeof(int16_t);      // A, P2, RK: [row][lane]
    static constexpr size_t PAT = (MAXM + 1 + 15) / 16 * 16;                            // pattern symbols, 1-based
    static constexpr size_t PER_WARP = PEQ + QUEUE + STATE + PAT;
    static_assert(PER_WARP % 16 == 0 && PER_WARP <= 227 * 1024, "DL state does not fit one warp's shared memory");
};

// Exact unrestricted Damerau-Levenshtein (Lowrance-Wagner, unit costs) of pat[1..m] against the lane's text (n symbols in the
// packed column src), streamed column by column over the text with O(m) state.  A transposition block whose gaps on both
// sides are >= 1 costs 1 + ga + gb >= 2 + max(ga, gb), which substitutions and indels already reach, so only two block shapes
// are needed (Zhao & Sahni 2019):
//   text gap 0    (a[i] = b[j-1]):  d[l-1][j-2] + (i - l),  l = last pattern row < i with a[l] = b[j]   -> L (register)
//   pattern gap 0 (a[i-1] = b[j]):  d[i-2][k-1] + (j - k),  k = last text column < j with b[k] = a[i]  -> RK[i] = d[i-2][k-1] - k
// A holds d[.][j-1] below row i and d[.][j] above it, P2 likewise d[.][j-2] / d[.][j-1]; both are stored relative to their
// column (d[r][c] - c lies in [-m, m]), so int16 fits every pattern length.  Rows are 32 lanes apart (conflict-free).
// Symbol 0 (text-only code points) equals nothing.
__device__ __forceinline__ int dl_dp(const uint8_t *__restrict__ pat, int m, const uint32_t *__restrict__ src, int n,
                                  int16_t *A, int16_t *P2, int16_t *RK) {
    if (m == 0) return n;
    for (int r = 0; r <= m; ++r) { A[r * 32] = (int16_t)r; P2[r * 32] = 0; RK[r * 32] = DL_NONE; }
    int bprev = 0, last = m;
    uint32_t word = 0;
    for (int j = 1; j <= n; ++j) {
        if (((j - 1) & 3) == 0) word = src[(size_t)((j - 1) >> 2) * 32];
        const int bj = (word >> (8 * ((j - 1) & 3))) & 0xff;
        int up = j, diag = j - 1, pdiag = 0, ap = 0;
        int L = 1 << 28;                                       // no row l < i with a[l] = b[j] yet
        for (int i = 1; i <= m; ++i) {
            const int ai = pat[i];
            const int left = A[i * 32] + (j - 1);
            const int p2 = P2[(i - 1) * 32] + (j - 2);
            const bool eq = bj != 0 && ai == bj;
            int d = min(diag + (eq ? 0 : 1), min(up, left) + 1);
            if (bprev != 0 && ai == bprev) d = min(d, L + i);
            if (ap != 0 && ap == bj) d = min(d, RK[i * 32] + j);
            if (eq) {
                L = p2 - i;
                if (i >= 2) RK[i * 32] = (int16_t)(pdiag - j);
            }
            P2[(i - 1) * 32] = (int16_t)(diag - (j - 1));
            A[i * 32] = (int16_t)(d - j);
            pdiag = diag; diag = left; up = d; ap = ai;
        }
        P2[m * 32] = (int16_t)(diag - (j - 1));
        bprev = bj;
        last = up;
    }
    return last;
}

template <typename W, int NW, int WARPS, bool TOPK>
__global__ void __launch_bounds__(WARPS * 32, 1) dl_kernel(const LevParams P, const double *__restrict__ gate) {
    constexpr int B = WordOps<W>::BITS;
    using Lay = DlLayout<W, NW>;
    extern __shared__ __align__(16) unsigned char dyn[];
    const int lane = lane_id();
    const int w = threadIdx.x >> 5;
    unsigned char *base = dyn + (size_t)w * Lay::PER_WARP;
    W *peq = reinterpret_cast<W *>(base);                                    // peq[sym * NW + block]
    int2 *queue = reinterpret_cast<int2 *>(base + Lay::PEQ);
    int16_t *sA = reinterpret_cast<int16_t *>(base + Lay::PEQ + Lay::QUEUE) + lane;
    int16_t *sP2 = sA + (Lay::MAXM + 1) * 32, *sRK = sP2 + (Lay::MAXM + 1) * 32;
    uint8_t *pat = base + Lay::PEQ + Lay::QUEUE + Lay::STATE;
    const bool norm = P.metric == PFZ_METRIC_NORM_DL;
    const bool full = P.matrix != nullptr;                                  // matrix mode: the DP on every pair
    const double NEG_INF = -CUDART_INF;
    const GroupRange gr = split_groups(P.n_to, P.n_splits);

    for (;;) {
        const int i = claim_row(P.counter + blockIdx.y, P.from_ids, P.n_ids);
        if (i < 0) break;
        const int64_t fb = P.from_off[i];
        const int m = (int)(P.from_off[i + 1] - fb);
        build_peq<W, NW>(peq, P.from_blob + fb, m, P.sym_table, pat);
        const int last_bit = (m - 1) & (B - 1);
        const int last_blk = m > 0 ? (m - 1) / B : 0;
        const double gt = gate ? gate[i] : NEG_INF;

        WarpArgBest<> best;
        WarpTopK top;
        if constexpr (TOPK) top.init(P.k); else best.init();
        double kth = NEG_INF;                                               // warp-uniform running k-th exact score
        int qn = 0;                                                         // warp-uniform queue fill

        auto score = [&](int d, int n) { return norm ? score_of(PFZ_METRIC_NORM_LEV, d, m, n) : -(double)d; };
        auto offer = [&](bool have, int d, int n, int orig) {
            double sc = 0.0; int cj = -1;
            if (have) {
                sc = score(d, n);
                const bool ok = !(P.exclude_self && (int64_t)orig == (int64_t)i + P.self_shift) && !(norm && !(sc >= P.cutoff));
                if (ok) cj = orig;
            }
            if constexpr (TOPK) {
                top.offer(sc, cj);
                const double ts = shfl_d(top.s, P.k - 1);
                kth = __shfl_sync(FULL, top.j, P.k - 1) >= 0 ? ts : NEG_INF;
            } else {
                best.offer(sc, cj, d);
                double v = best.j >= 0 ? best.s : NEG_INF;
#pragma unroll
                for (int o = 16; o; o >>= 1) v = fmax(v, shfl_d(v, lane ^ o));
                kth = v;
            }
        };
        // all lanes: lane r < cnt takes queue entry r, re-tests it against the threshold (which may have risen since it was
        // queued) and runs the DP
        auto flush = [&](int cnt) {
            const bool act = lane < cnt;
            const int2 e = act ? queue[lane] : make_int2(0, 0);
            const int n = act ? P.slen[e.x] : 0;
            const int orig = act ? P.sorig[e.x] : -1;
            const bool run = act && (full || !(score(e.y, n) < fmax(gt, kth)));
            int d = 0;
            if (run) d = dl_dp(pat, m, P.packed + P.grp_word_off[e.x >> 5] + (e.x & 31), n, sA, sP2, sRK);
            if (run && full) P.matrix[(int64_t)i * P.matrix_ld + orig] = d;
            offer(run, d, n, orig);
        };

        for (int g = gr.lo; g < gr.hi; ++g) {
            const int p = g * 32 + lane;
            const bool have = p < P.n_to;
            const int n = have ? P.slen[p] : 0;
            const int orig = have ? P.sorig[p] : -1;
            const uint32_t *src = P.packed + P.grp_word_off[g] + lane;
            LevColumn<W, NW, true> col;
            col.init();
            int score_m = m;
            for_each_text_symbol(src, n, [&](int s) { score_m += col.step(peq + s * NW, last_blk, last_bit); });
            const int osa = m > 0 ? score_m : n;
            const int lb = max((2 * osa + 2) / 3, abs(m - n));
            const bool excl = P.exclude_self && (int64_t)orig == (int64_t)i + P.self_shift;
            bool direct = false, queued = false;
            if (have && full) queued = true;
            else if (have && !excl) {
                const double ub = score(lb, n);
                if (!(ub < fmax(gt, kth)) && !(norm && ub < P.cutoff)) {
                    if (lb == osa) direct = true; else queued = true;
                }
            }
            if (__any_sync(FULL, direct)) offer(direct, osa, n, orig);
            const unsigned need = __ballot_sync(FULL, queued);
            if (need) {
                const int pos = qn + __popc(need & ((1u << lane) - 1u));
                if (queued && pos < 32) queue[pos] = make_int2(p, lb);
                int tot = qn + __popc(need);
                if (tot >= 32) {
                    __syncwarp();
                    flush(32);
                    __syncwarp();
                    if (queued && pos >= 32) queue[pos - 32] = make_int2(p, lb);
                    tot -= 32;
                }
                qn = tot;
                __syncwarp();
            }
        }
        if (qn > 0) flush(qn);

        store_row<TOPK>(P, i, top, best);
        __syncwarp();
    }
}

template <typename W, int NW> struct WordClass { using Word = W; static constexpr int N = NW; };

// n_words (0: one 32-bit word; 1, 2, 4, 8, 16 64-bit words) -> f(WordClass<W, NW>())
template <typename F>
static int dispatch_words(int n_words, F &&f) {
    switch (n_words) {
        case 0: return f(WordClass<uint32_t, 1>());
        case 1: return f(WordClass<uint64_t, 1>());
        case 2: return f(WordClass<uint64_t, 2>());
        case 4: return f(WordClass<uint64_t, 4>());
        case 8: return f(WordClass<uint64_t, 8>());
        default: return f(WordClass<uint64_t, 16>());
    }
}

// word class -> kernel instantiation; the metric picks Levenshtein, Indel, OSA, Jaro or DL (gate: DL only)
template <bool TOPK>
static int launch_class(const LevParams &P, const double *gate, int n_words, int sms, cudaStream_t st) {
    const int mt = P.metric;
    return dispatch_words(n_words, [&](auto c) {
        using W = typename decltype(c)::Word;
        constexpr int NW = decltype(c)::N;
        if (mt == PFZ_METRIC_DL || mt == PFZ_METRIC_NORM_DL) {
            // Shared memory per warp (DlLayout): 7.6 KB at 32 symbols, 15 KB at 64, ..., 225 KB at 1 024 -- 4 warps per CTA up
            // to 256 symbols, 2 at 512, 1 at 1 024.
            constexpr size_t PER_WARP = DlLayout<W, NW>::PER_WARP;
            constexpr int WARPS = warps_within(PER_WARP, 227 * 1024);
            return launch_rows(dl_kernel<W, NW, WARPS, TOPK>, WARPS, WARPS * PER_WARP, P.n_ids, P.n_splits, sms, st, P, gate);
        }
        if (mt == PFZ_METRIC_JARO || mt == PFZ_METRIC_JARO_WINKLER) {
            // Shared memory per warp: Peq (256 x NW words) plus the match store (32 lanes x B*NW bytes), the same size again.
            // Up to 64 KB per CTA: 4 warps up to 256 code points, 2 at 512, 1 at 1 024.
            constexpr size_t PER_WARP = 2 * 256 * NW * sizeof(W);
            constexpr int WARPS = warps_within(PER_WARP, 65536);
            return launch_rows(jaro_kernel<W, NW, WARPS, TOPK>, WARPS, WARPS * PER_WARP, P.n_ids, P.n_splits, sms, st, P);
        }
        constexpr int WARPS = 4;
        const size_t smem = (size_t)WARPS * 256 * NW * sizeof(W);
        if (mt == PFZ_METRIC_OSA || mt == PFZ_METRIC_NORM_OSA)
            return launch_rows(lev_kernel<W, NW, false, WARPS, TOPK, true>, WARPS, smem, P.n_ids, P.n_splits, sms, st, P);
        if (mt == PFZ_METRIC_INDEL || mt == PFZ_METRIC_RATIO)
            return launch_rows(lev_kernel<W, NW, true, WARPS, TOPK>, WARPS, smem, P.n_ids, P.n_splits, sms, st, P);
        return launch_rows(lev_kernel<W, NW, false, WARPS, TOPK>, WARPS, smem, P.n_ids, P.n_splits, sms, st, P);
    });
}

// The body of the four K3 entry points after their metric checks: the checks they share, the row counters and the launch.
// fn names the entry point in error messages.
template <bool TOPK>
static int run_k3(const char *fn, const uint32_t *from_blob, const int64_t *from_offsets, int32_t n_from, const int32_t *from_ids,
                  int32_t n_ids, int32_t n_words, const uint8_t *sym_table, const uint32_t *packed, const int64_t *grp_word_off,
                  const int32_t *slen, const int32_t *sorig, int32_t n_to, int32_t metric, double score_cutoff, int32_t exclude_self,
                  int64_t self_shift, int32_t n_splits, int32_t k, int32_t *part_idx, double *part_score, int32_t *part_dist,
                  int32_t *matrix, int64_t matrix_ld, const double *gate, int32_t *counter, void *stream) {
    PFZ_REQUIRE(n_words == 0 || n_words == 1 || n_words == 2 || n_words == 4 || n_words == 8 || n_words == 16,
                "%s: n_words %d unsupported (0 = 32-bit word, 1, 2, 4, 8, 16 64-bit words)", fn, n_words);
    PFZ_REQUIRE(n_splits >= 1, "%s: n_splits < 1", fn);
    PFZ_REQUIRE(!TOPK || (k >= 1 && k <= 32), "%s: k=%d unsupported (1..32)", fn, k);
    if (n_ids <= 0 || n_to < 0) return 0;
    cudaStream_t st = as_stream(stream);
    int sms = 0;
    if (start_rows(counter, n_splits, st, &sms)) return 1;
    LevParams P{from_blob, from_offsets, from_ids, n_ids, sym_table, packed, grp_word_off, slen, sorig, n_to, metric, score_cutoff,
                exclude_self, self_shift, ratio_min_ns_of(score_cutoff), n_splits, part_idx, part_score, part_dist, matrix, matrix_ld, n_from,
                counter, k};
    return launch_class<TOPK>(P, gate, n_words, sms, st);
}

}  // namespace pfz

using namespace pfz;

extern "C" {

int pfz_lev_pack(const uint32_t *to_blob, const int64_t *to_offsets, const int32_t *order, int32_t n_to, const uint8_t *sym_table,
                 const int64_t *grp_word_off, uint32_t *packed, int32_t *slen, void *stream) {
    if (n_to <= 0) return 0;
    const int n_grp = (n_to + 31) / 32;
    int grid = (n_grp + 7) / 8; if (grid > SM_COUNT * 8) grid = SM_COUNT * 8;
    lev_pack_kernel<<<grid, 256, 0, as_stream(stream)>>>(to_blob, to_offsets, order, n_to, sym_table, grp_word_off, packed, slen);
    PFZ_LAUNCH_OK();
    return 0;
}

int pfz_lev_argbest(const uint32_t *from_blob, const int64_t *from_offsets, int32_t n_from, const int32_t *from_ids, int32_t n_ids,
                    int32_t n_words, const uint8_t *sym_table, const uint32_t *packed, const int64_t *grp_word_off, const int32_t *slen,
                    const int32_t *sorig, int32_t n_to, int32_t metric, double score_cutoff, int32_t exclude_self, int64_t self_shift,
                    int32_t n_splits, int32_t *part_idx, double *part_score, int32_t *part_dist, int32_t *matrix, int64_t matrix_ld,
                    int32_t *counter, void *stream) {
    PFZ_REQUIRE(metric >= PFZ_METRIC_LEV && metric <= PFZ_METRIC_NORM_OSA, "pfz_lev_argbest: unknown metric %d", metric);
    const bool jaro = metric == PFZ_METRIC_JARO || metric == PFZ_METRIC_JARO_WINKLER;
    PFZ_REQUIRE(!(jaro && matrix), "pfz_lev_argbest: the distance matrix is not available for the Jaro metrics (matrix must be NULL)");
    return run_k3<false>("pfz_lev_argbest", from_blob, from_offsets, n_from, from_ids, n_ids, n_words, sym_table, packed, grp_word_off,
                         slen, sorig, n_to, metric, score_cutoff, exclude_self, self_shift, n_splits, 1, part_idx, part_score, part_dist,
                         matrix, matrix_ld, nullptr, counter, stream);
}

int pfz_lev_topk(const uint32_t *from_blob, const int64_t *from_offsets, int32_t n_from, const int32_t *from_ids, int32_t n_ids,
                 int32_t n_words, const uint8_t *sym_table, const uint32_t *packed, const int64_t *grp_word_off, const int32_t *slen,
                 const int32_t *sorig, int32_t n_to, int32_t metric, double score_cutoff, int32_t exclude_self, int64_t self_shift,
                 int32_t n_splits, int32_t k, int32_t *part_idx, double *part_score, int32_t *counter, void *stream) {
    PFZ_REQUIRE((metric >= PFZ_METRIC_NORM_LEV && metric <= PFZ_METRIC_JARO_WINKLER) || metric == PFZ_METRIC_NORM_OSA,
                "pfz_lev_topk: metric %d unsupported (NORM_LEV, RATIO, JARO, JARO_WINKLER, NORM_OSA)", metric);
    return run_k3<true>("pfz_lev_topk", from_blob, from_offsets, n_from, from_ids, n_ids, n_words, sym_table, packed, grp_word_off,
                        slen, sorig, n_to, metric, score_cutoff, exclude_self, self_shift, n_splits, k, part_idx, part_score, nullptr,
                        nullptr, 0, nullptr, counter, stream);
}

int pfz_dl_argbest(const uint32_t *from_blob, const int64_t *from_offsets, int32_t n_from, const int32_t *from_ids, int32_t n_ids,
                   int32_t n_words, const uint8_t *sym_table, const uint32_t *packed, const int64_t *grp_word_off, const int32_t *slen,
                   const int32_t *sorig, int32_t n_to, int32_t metric, double score_cutoff, int32_t exclude_self, int64_t self_shift,
                   int32_t n_splits, int32_t *part_idx, double *part_score, int32_t *part_dist, int32_t *matrix, int64_t matrix_ld,
                   const double *gate, int32_t *counter, void *stream) {
    PFZ_REQUIRE(metric == PFZ_METRIC_DL || metric == PFZ_METRIC_NORM_DL, "pfz_dl_argbest: metric %d unsupported (DL, NORM_DL)", metric);
    PFZ_REQUIRE(!(matrix && gate), "pfz_dl_argbest: the distance matrix needs every pair, so gate must be NULL with a matrix");
    return run_k3<false>("pfz_dl_argbest", from_blob, from_offsets, n_from, from_ids, n_ids, n_words, sym_table, packed, grp_word_off,
                         slen, sorig, n_to, metric, score_cutoff, exclude_self, self_shift, n_splits, 1, part_idx, part_score, part_dist,
                         matrix, matrix_ld, gate, counter, stream);
}

int pfz_dl_topk(const uint32_t *from_blob, const int64_t *from_offsets, int32_t n_from, const int32_t *from_ids, int32_t n_ids,
                int32_t n_words, const uint8_t *sym_table, const uint32_t *packed, const int64_t *grp_word_off, const int32_t *slen,
                const int32_t *sorig, int32_t n_to, int32_t metric, double score_cutoff, int32_t exclude_self, int64_t self_shift,
                int32_t n_splits, int32_t k, int32_t *part_idx, double *part_score, const double *gate, int32_t *counter, void *stream) {
    PFZ_REQUIRE(metric == PFZ_METRIC_NORM_DL, "pfz_dl_topk: metric %d unsupported (NORM_DL)", metric);
    return run_k3<true>("pfz_dl_topk", from_blob, from_offsets, n_from, from_ids, n_ids, n_words, sym_table, packed, grp_word_off,
                        slen, sorig, n_to, metric, score_cutoff, exclude_self, self_shift, n_splits, k, part_idx, part_score, nullptr,
                        nullptr, 0, gate, counter, stream);
}

int pfz_lev_merge(const int32_t *part_idx, const double *part_score, const int32_t *part_dist, int32_t n_splits, int32_t n_from,
                  int32_t *best_idx, double *best_score, int32_t *best_dist, void *stream) {
    if (n_from <= 0) return 0;
    int grid = (n_from + 255) / 256; if (grid > SM_COUNT * 8) grid = SM_COUNT * 8;
    lev_merge_kernel<<<grid, 256, 0, as_stream(stream)>>>(part_idx, part_score, part_dist, n_splits, n_from, best_idx, best_score, best_dist);
    PFZ_LAUNCH_OK();
    return 0;
}
}
