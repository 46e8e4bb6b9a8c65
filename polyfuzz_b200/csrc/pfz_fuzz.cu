// pfz_fuzz.cu -- K3b: rapidfuzz's token / partial / weighted scorers over the |from| x |to| grid with a fused per-row
// arg-best (process.extractOne semantics: the first to-string with the maximal score >= score_cutoff).
//
// Replaces the scorer loop of the reference's edit-distance matchers for the scorers beyond fuzz.ratio:
//     polyfuzz/models/_rapidfuzz.py:48       scorer=fuzz.WRatio, the default of RapidFuzz and of PolyFuzz("EditDistance")
//     polyfuzz/models/_rapidfuzz.py:24-37    partial_ratio, token_sort_ratio, token_set_ratio, token_ratio, partial_token_*, QRatio
//     polyfuzz/models/_rapidfuzz.py:106-108  process.extractOne(query, to_list, scorer=..., score_cutoff=...)
// The scorer definitions (incl. the order of the double-precision operations and the way score_cutoff is threaded through
// WRatio) are those of rapidfuzz 3.x as restated and pinned on rapidfuzz's published known answers in oracle/fuzz.py.
//
// Mapping (as K3, pfz_lev.cu, and with its row driver from pfz_common.cuh): one warp = one from-string, whose bit-vector match masks Peq[symbol] live in shared memory
// for THREE derived patterns -- a itself, S(a) = its whitespace tokens sorted and joined, U(a) = its distinct tokens sorted and
// joined; one lane = one to-string at a time (to-strings pre-sorted by length, groups of 32, transposed, 4 byte-symbols per
// word), with the same three variants b, S(b), U(b).  Every Indel distance is a bit-parallel LCS (Hyyro 2004):
//   ratio                LCS(a, b)
//   token_sort_ratio     LCS(S(a), S(b))
//   token_set_ratio      token-id sets (sorted ids per string, 64-bit Bloom signature as a pre-filter): no common token ->
//                        LCS(U(a), U(b)); a common token and one side a subset -> 100; else the differences are joined per
//                        pair and scored by a masked LCS over U(a)'s bits (fz_diff_indel)
//   partial_ratio        the shorter string against every window of the longer one (prefixes shorter than it, all windows of
//                        its length, suffixes): windows of the to-string restart the recurrence at the window start; windows of
//                        the from-string mask Peq to the window's bits; prefix windows fall out of ONE pass (the number of zero
//                        bits among the first i rows is LCS(a[:i], b))
//   WRatio               the weighted combination (0.95 / 0.9 / 0.6, length-ratio switches 1.5 and 8) of the above.
// Symbols are bytes (the host maps the code points of the from-list to 1..255, everything else to 0 = matches nothing).
//
// Word classes: NW = 1, 2, 4 (from-strings up to 256 code points) run one warp per from-row, WARPS warps per CTA, each warp
// with its own masks of the three variants.  NW = 8, 16 (257..1 024) run one CTA per from-row (CTA_ROW): the CTA's warps share
// the masks of the variants the scorer reads and take the split's to-groups in turn; their epilogues are merged at the end of
// the row (merge_cta).  To-strings may have any length.
#include "pfz_common.cuh"

namespace pfz {

enum { FZ_RATIO = 0, FZ_QRATIO = 1, FZ_PARTIAL = 2, FZ_TSORT = 3, FZ_TSET = 4, FZ_TRATIO = 5, FZ_PTSORT = 6, FZ_PTSET = 7, FZ_PTRATIO = 8, FZ_WRATIO = 9 };

struct FuzzSide {                       // one string list with its derived variants (device pointers)
    const uint32_t *blob[3]; const int64_t *off[3];         // UTF-32 code points + offsets of s, S(s), U(s)
    const int32_t *tok_ptr; const int32_t *tok_ids;         // distinct token ids per string, ascending
    const uint64_t *sig;                                    // Bloom signature of the token ids
    const int32_t *n_tok_all;                               // number of tokens incl. duplicates
};
struct FuzzParams {
    FuzzSide F;                                             // from-strings (patterns)
    FuzzSide T;                                             // to-strings: blobs used by the per-pair slow path only
    const int32_t *from_ids; int n_ids;                     // from-rows of this word class
    const uint8_t *sym_table;
    const uint32_t *packed[3]; const int64_t *grp_off[3]; const int32_t *slen[3];   // to-side transposed layouts of b, S(b), U(b)
    const int32_t *sorig; int n_to;
    const uint32_t *tok_blob; const int64_t *tok_off;       // token texts (code points) by token id
    int scorer; double cutoff; int exclude_self; int64_t self_shift;
    int n_splits; int32_t *part_idx; double *part_score; int n_from; int32_t *counter;
    int k;                                                  // top-k epilogue: list length; part_* are [n_splits][n_from][k]
};

// ---- scalar scorer algebra (double, no contraction) -- mirrors oracle/fuzz.py line by line -------------------------------------
__device__ __forceinline__ double fz_norm_sim(int dist, int lensum) {          // Indel.normalized_similarity
    const double nd = lensum ? __ddiv_rn((double)dist, (double)lensum) : 0.0;
    return __dsub_rn(1.0, nd);
}
__device__ __forceinline__ double fz_ratio(int lcs, int la, int lb, double cutoff) {
    const double ns = fz_norm_sim(la + lb - 2 * lcs, la + lb);
    return ns >= __ddiv_rn(cutoff, 100.0) ? __dmul_rn(ns, 100.0) : 0.0;
}
__device__ __forceinline__ double fz_norm_distance(int dist, int lensum, double cutoff) {
    const double sc = lensum ? __dsub_rn(100.0, __ddiv_rn(__dmul_rn(100.0, (double)dist), (double)lensum)) : 100.0;
    return sc >= cutoff ? sc : 0.0;
}
// partial_ratio's two cutoff steps: its windows are scored at cutoff / 100 (best_ns is kept only if best_ns >= cutoff / 100),
// then the result best_ns * 100 only if it is >= cutoff -- as fz_ratio, they disagree whenever (ns * 100) / 100 != ns
__device__ __forceinline__ double fz_partial_from_best(double best_ns, bool both_empty, double cutoff) {
    if (both_empty) return 100.0;
    const double res = __dmul_rn(best_ns, 100.0);
    return best_ns >= __ddiv_rn(cutoff, 100.0) && res >= cutoff ? res : 0.0;
}

// ---- bit-parallel LCS over NW 64-bit blocks ------------------------------------------------------------------------------------
template <int NW>
struct Bp {
    uint64_t S[NW];
    __device__ __forceinline__ void init() {
#pragma unroll
        for (int b = 0; b < NW; ++b) S[b] = ~0ull;
    }
    // one text symbol; mask (may be null) restricts the pattern to a window of its rows
    __device__ __forceinline__ void step(const uint64_t *__restrict__ peq, int s, const uint64_t *mask) {
        unsigned carry = 0;
#pragma unroll
        for (int b = 0; b < NW; ++b) {
            uint64_t Eq = peq[s * NW + b];
            if (mask) Eq &= mask[b];
            const uint64_t x = S[b], u = x & Eq;
            const uint64_t sum = x + u; unsigned c1 = sum < x; const uint64_t sum2 = sum + carry; c1 |= (sum2 < sum); carry = c1;
            S[b] = sum2 | (x & ~Eq);
        }
    }
    // LCS(pattern[lo:hi), text so far): zero bits among rows lo..hi-1
    __device__ __forceinline__ int zeros(int lo, int hi) const {
        int z = 0;
#pragma unroll
        for (int b = 0; b < NW; ++b) {
            const int l = max(lo - 64 * b, 0), h = min(hi - 64 * b, 64);
            if (h > l) {
                uint64_t m = (h == 64 ? ~0ull : ((1ull << h) - 1ull)) & ~((1ull << l) - 1ull);
                z += __popcll(~S[b] & m);
            }
        }
        return z;
    }
};

struct TextRef { const uint32_t *src; int n; };           // lane-strided packed words of one to-string variant
__device__ __forceinline__ int text_sym(const TextRef &t, int j) { return (t.src[(size_t)(j >> 2) * 32] >> (8 * (j & 3))) & 0xff; }

template <int NW>
__device__ int fz_lcs(const uint64_t *__restrict__ peq, int m, const TextRef &t) {
    if (m == 0 || t.n == 0) return 0;
    Bp<NW> bp; bp.init();
    for (int j = 0; j < t.n; ++j) bp.step(peq, text_sym(t, j), nullptr);
    return bp.zeros(0, m);
}

// best normalised Indel similarity of partial_ratio(pattern, text): rapidfuzz's window set (see the file header).
// SKIP (the long classes): a window whose boundary symbol -- the last one of a full window, the first one of a suffix -- does
// not occur in the other string is not scored.  It is dominated by a scored neighbour (DESIGN §4.3), so the best is unchanged.
template <int NW, bool SKIP = false>
__device__ double fz_partial_best(const uint64_t *__restrict__ peq, int la, const TextRef &t) {
    const int lb = t.n;
    double best = 0.0;
    if (la == 0 || lb == 0) return 0.0;                    // (both empty is handled by the caller)
    if (la <= lb) {                                        // shorter = pattern; windows of the text
        const int ls = la, ll = lb;
        Bp<NW> bp; bp.init();
        for (int j = 0; j + 1 < ls; ++j) {                 // prefixes text[:j+1], one pass
            bp.step(peq, text_sym(t, j), nullptr);
            best = fmax(best, fz_norm_sim(ls + (j + 1) - 2 * bp.zeros(0, ls), ls + j + 1));
        }
        for (int i = 0; i < ll; ++i) {                     // windows text[i : i+ls] (i < ll-ls) and suffixes text[i:] (i >= ll-ls)
            const int e = min(ll, i + ls);
            if constexpr (SKIP) {
                const int s = text_sym(t, i < ll - ls ? e - 1 : i);
                uint64_t any = 0;
#pragma unroll
                for (int b = 0; b < NW; ++b) any |= peq[s * NW + b];
                if (!any) continue;
            }
            bp.init();
            for (int j = i; j < e; ++j) bp.step(peq, text_sym(t, j), nullptr);
            best = fmax(best, fz_norm_sim(ls + (e - i) - 2 * bp.zeros(0, ls), ls + (e - i)));
        }
    }
    if (la > lb || (la == lb && best != 1.0)) {            // shorter = text; windows of the pattern
        const int ls = lb, ll = la;
        Bp<NW> bp; bp.init();
        uint64_t hit[SKIP ? NW : 1];                       // SKIP: the pattern rows whose symbol occurs in the text
        if constexpr (SKIP) {
#pragma unroll
            for (int b = 0; b < NW; ++b) hit[b] = 0;
        }
        for (int j = 0; j < ls; ++j) {
            const int s = text_sym(t, j);
            bp.step(peq, s, nullptr);
            if constexpr (SKIP) {
#pragma unroll
                for (int b = 0; b < NW; ++b) hit[b] |= peq[s * NW + b];
            }
        }
        for (int i = 1; i < ls; ++i)                       // prefixes pattern[:i]: rows 0..i-1 of the final state
            best = fmax(best, fz_norm_sim(ls + i - 2 * bp.zeros(0, i), ls + i));
        for (int i = 0; i < ll; ++i) {                     // windows pattern[i : i+ls] and suffixes pattern[i:]
            const int e = min(ll, i + ls);
            if constexpr (SKIP) {
                const int r = i < ll - ls ? e - 1 : i;
                uint64_t hw = 0;
#pragma unroll
                for (int b = 0; b < NW; ++b) hw = b == (r >> 6) ? hit[b] : hw;
                if (!((hw >> (r & 63)) & 1ull)) continue;
            }
            uint64_t mask[NW];
#pragma unroll
            for (int b = 0; b < NW; ++b) {
                const int l = max(i - 64 * b, 0), h = min(e - 64 * b, 64);
                mask[b] = (h > l) ? ((h == 64 ? ~0ull : ((1ull << h) - 1ull)) & ~((1ull << l) - 1ull)) : 0ull;
            }
            bp.init();
            for (int j = 0; j < ls; ++j) bp.step(peq, text_sym(t, j), mask);
            best = fmax(best, fz_norm_sim(ls + (e - i) - 2 * bp.zeros(i, e), ls + (e - i)));
        }
    }
    return best;
}

// ---- token sets ----------------------------------------------------------------------------------------------------------------
struct TokInfo { int n_common; int sect_len; int ab_len; int ba_len; int n_ab; int n_ba; };
// merge of the two ascending id lists: |intersection| and the joined lengths of intersection / differences (tokens + single spaces)
__device__ TokInfo fz_tok_info(const int32_t *a, int na, const int32_t *b, int nb, const int64_t *__restrict__ tok_off) {
    TokInfo r{0, 0, 0, 0, 0, 0};
    int p = 0, q = 0, sect = 0, ab = 0, ba = 0;
    while (p < na || q < nb) {
        const int x = p < na ? a[p] : 0x7fffffff, y = q < nb ? b[q] : 0x7fffffff;
        if (x == y) { sect += (int)(tok_off[x + 1] - tok_off[x]); ++r.n_common; ++p; ++q; }
        else if (x < y) { ab += (int)(tok_off[x + 1] - tok_off[x]); ++r.n_ab; ++p; }
        else { ba += (int)(tok_off[y + 1] - tok_off[y]); ++r.n_ba; ++q; }
    }
    r.sect_len = sect + max(r.n_common - 1, 0);
    r.ab_len = ab + max(r.n_ab - 1, 0);
    r.ba_len = ba + max(r.n_ba - 1, 0);
    return r;
}
// Indel distance of the joined differences (tokens of a not in b, sorted | tokens of b not in a, sorted) as a bit-parallel LCS
// over U(a)'s masks.  U(a) is a's distinct tokens in id order (= sorted order: the host numbers the tokens in sorted order)
// joined by single spaces, so the from-side difference is the subsequence of U(a) made of its kept tokens and the space
// before every kept token but the first.  The other rows are masked off: they never match, so the LCS against them is the
// LCS against the difference.  The to-side difference is streamed from tok_blob (with its spaces) as the text; a code point
// outside the alphabet maps to 0 and matches nothing.  No per-thread arrays; the text has any length.
__device__ __forceinline__ int fz_sym(uint32_t c, const uint8_t *__restrict__ sym_table) { return c < 0x110000u ? sym_table[c] : 0; }

template <int NW>
__device__ int fz_diff_indel(const uint64_t *__restrict__ peq_u, const int32_t *a, int na, const int32_t *b, int nb,
                             const uint32_t *__restrict__ tok_blob, const int64_t *__restrict__ tok_off, const uint8_t *__restrict__ sym_table) {
    uint64_t mask[NW];
#pragma unroll
    for (int w = 0; w < NW; ++w) mask[w] = 0;
    int la = 0;
    for (int p = 0, q = 0, pos = 0; p < na; ++p) {         // a \ b: rows of U(a) kept
        const int x = a[p];
        while (q < nb && b[q] < x) ++q;
        const int len = (int)(tok_off[x + 1] - tok_off[x]);
        if (q >= nb || b[q] != x) {
            const int l = la ? pos - 1 : pos, h = pos + len;
            la += h - l;
#pragma unroll
            for (int w = 0; w < NW; ++w) {
                const int lo = max(l - 64 * w, 0), hi = min(h - 64 * w, 64);
                if (hi > lo) mask[w] |= (hi == 64 ? ~0ull : ((1ull << hi) - 1ull)) & ~((1ull << lo) - 1ull);
            }
        }
        pos += len + 1;
    }
    const int space = sym_table[0x20];
    Bp<NW> bp; bp.init();
    int lb = 0;
    for (int p = 0, q = 0; q < nb; ++q) {                  // b \ a, streamed
        const int y = b[q];
        while (p < na && a[p] < y) ++p;
        if (p < na && a[p] == y) continue;
        if (lb) { bp.step(peq_u, space, mask); ++lb; }
        for (int64_t c = tok_off[y]; c < tok_off[y + 1]; ++c, ++lb) bp.step(peq_u, fz_sym(tok_blob[c], sym_table), mask);
    }
    return la + lb - 2 * bp.zeros(0, 64 * NW);
}

// TOPK = false: per-row arg-best; TOPK = true: the k best per row in a WarpTopK, offered after every group of 32 to-strings
// (the group's body is a do/while(0), so a lane that skips its pair still reaches the warp-wide offer).
// (minimum 1 block per SM for TOPK: without it ptxas's register target makes some top-k classes spill; for the arg-best
// classes at 1 and 2 words, the blocks per SM their shared memory and registers allow, which keeps ptxas from spilling more)
// CTA_ROW (NW >= 8): dyn holds the masks of the variants the scorer reads (fz_variants), in variant order, then the merge
// buffers and the row slot (fz_cta_smem).
__host__ __device__ constexpr bool fz_reads_plain(int sc) { return sc == FZ_RATIO || sc == FZ_QRATIO || sc == FZ_PARTIAL || sc == FZ_WRATIO; }
__host__ __device__ constexpr bool fz_reads_sorted(int sc) { return sc == FZ_TSORT || sc == FZ_TRATIO || sc == FZ_PTSORT || sc == FZ_PTRATIO || sc == FZ_WRATIO; }
__host__ __device__ constexpr bool fz_reads_uniq(int sc) { return sc == FZ_TSET || sc == FZ_TRATIO || sc == FZ_PTSET || sc == FZ_PTRATIO || sc == FZ_WRATIO; }
__host__ __device__ constexpr int fz_variants(int sc) { return (int)fz_reads_plain(sc) + (int)fz_reads_sorted(sc) + (int)fz_reads_uniq(sc); }
constexpr size_t fz_cta_smem(int nw, int warps, int sc) { return (size_t)fz_variants(sc) * 256 * nw * 8 + (size_t)warps * 32 * 12 + 16; }

template <int NW, int WARPS, bool TOPK = false>
__global__ void __launch_bounds__(WARPS * 32, TOPK ? 1 : NW == 1 ? 6 : NW == 2 ? 9 : 0) fuzz_kernel(const FuzzParams P) {
    constexpr bool CTA_ROW = NW >= 8;
    extern __shared__ __align__(16) unsigned char dyn[];
    const int lane = lane_id();
    const int w = threadIdx.x >> 5;
    const int sc_id = P.scorer;
    const bool need_sorted = fz_reads_sorted(sc_id), need_uniq = fz_reads_uniq(sc_id);
    uint64_t *peq_all = nullptr;                                     // one warp: peq[variant][sym * NW + block]
    uint64_t *peq_v[3];                                    // CTA_ROW: the variants the scorer reads, packed
    double *sh_s = nullptr; int *sh_j = nullptr, *slot = nullptr;
    if constexpr (CTA_ROW) {
        peq_v[0] = reinterpret_cast<uint64_t *>(dyn);
        peq_v[1] = peq_v[0] + (fz_reads_plain(sc_id) ? 256 * NW : 0);
        peq_v[2] = peq_v[1] + (need_sorted ? 256 * NW : 0);
        sh_s = reinterpret_cast<double *>(peq_v[2] + (need_uniq ? 256 * NW : 0));
        sh_j = reinterpret_cast<int *>(sh_s + WARPS * 32);
        slot = sh_j + WARPS * 32;
    } else {
        peq_all = reinterpret_cast<uint64_t *>(dyn) + (size_t)w * 3 * 256 * NW;
    }

    for (;;) {
        int i;
        if constexpr (CTA_ROW) i = claim_row_cta(P.counter + blockIdx.y, P.from_ids, P.n_ids, slot);
        else i = claim_row(P.counter + blockIdx.y, P.from_ids, P.n_ids);
        if (i < 0) break;
        const GroupRange gr = split_groups(P.n_to, P.n_splits);    // per row: held across rows, it adds spills (2 words)
        int lens[3];
        for (int v = 0; v < 3; ++v) {
            const int64_t fb = P.F.off[v][i];
            lens[v] = (int)(P.F.off[v][i + 1] - fb);
            if ((v == 1 && !need_sorted) || (v == 2 && !need_uniq)) continue;
            if constexpr (CTA_ROW) {
                if (v == 0 && !fz_reads_plain(sc_id)) continue;
                build_peq<uint64_t, NW, true>(peq_v[v], P.F.blob[v] + fb, lens[v], P.sym_table);
            } else {
                build_peq<uint64_t, NW>(peq_all + (size_t)v * 256 * NW, P.F.blob[v] + fb, lens[v], P.sym_table);
            }
        }
        const int la = lens[0], las = lens[1], lau = lens[2];
        const int32_t *atok = P.F.tok_ids + P.F.tok_ptr[i];
        const int na = P.F.tok_ptr[i + 1] - P.F.tok_ptr[i];
        const int na_all = P.F.n_tok_all[i];
        const uint64_t asig = P.F.sig[i];
        const uint64_t *peq0, *peq1, *peq2;
        if constexpr (CTA_ROW) { peq0 = peq_v[0]; peq1 = peq_v[1]; peq2 = peq_v[2]; }
        else { peq0 = peq_all; peq1 = peq_all + 256 * NW; peq2 = peq_all + 2 * 256 * NW; }

        WarpArgBest<false> best;
        WarpTopK top;
        if constexpr (TOPK) top.init(P.k); else best.init();
        for (int g = gr.lo + (CTA_ROW ? w : 0); g < gr.hi; g += CTA_ROW ? WARPS : 1) {
            double cand_s = 0.0; int cand_j = -1;
            do {
                const int p = g * 32 + lane;
                if (p >= P.n_to) continue;
                const int orig = P.sorig[p];
                if (P.exclude_self && (int64_t)orig == (int64_t)i + P.self_shift) continue;
                TextRef t0{P.packed[0] + P.grp_off[0][g] + lane, P.slen[0][p]};
                TextRef t1{P.packed[1] + P.grp_off[1][g] + lane, P.slen[1][p]};
                TextRef t2{P.packed[2] + P.grp_off[2][g] + lane, P.slen[2][p]};
                const int lb = t0.n;
                const double cut = P.cutoff;
                // token-set facts of the pair, computed on demand
                bool tok_done = false; TokInfo ti{0, 0, 0, 0, 0, 0};
                const int32_t *btok = P.T.tok_ids + P.T.tok_ptr[orig];
                const int nb = P.T.tok_ptr[orig + 1] - P.T.tok_ptr[orig];
                const int nb_all = P.T.n_tok_all[orig];
                auto tok = [&]() {
                    if (!tok_done) {
                        if ((asig & P.T.sig[orig]) == 0ull) {   // no common token possible: differences are the whole distinct-token strings
                            ti.n_common = 0; ti.sect_len = 0; ti.ab_len = lau; ti.ba_len = t2.n; ti.n_ab = na; ti.n_ba = nb;
                        } else ti = fz_tok_info(atok, na, btok, nb, P.tok_off);
                        tok_done = true;
                    }
                };
                auto token_sort = [&](double c) { return fz_ratio(fz_lcs<NW>(peq1, las, t1), las, t1.n, c); };
                auto token_set = [&](double c) -> double {
                    if (c > 100.0) return 0.0;
                    if (na == 0 || nb == 0) return 0.0;
                    tok();
                    if (ti.n_common && (ti.n_ab == 0 || ti.n_ba == 0)) return 100.0;
                    const int sect_len = ti.sect_len;
                    const int sect_ab_len = sect_len + (sect_len != 0) + ti.ab_len;
                    const int sect_ba_len = sect_len + (sect_len != 0) + ti.ba_len;
                    double result = 0.0;
                    const double cd = ceil(__dmul_rn((double)(sect_ab_len + sect_ba_len), __dsub_rn(1.0, __ddiv_rn(c, 100.0))));
                    const int dist = ti.n_common == 0 ? (lau + t2.n - 2 * fz_lcs<NW>(peq2, lau, t2))
                                                      : fz_diff_indel<NW>(peq2, atok, na, btok, nb, P.tok_blob, P.tok_off, P.sym_table);
                    if ((double)dist <= cd) result = fz_norm_distance(dist, sect_ab_len + sect_ba_len, c);
                    if (!sect_len) return result;
                    const double r_ab = fz_norm_distance((sect_len != 0) + ti.ab_len, sect_len + sect_ab_len, c);
                    const double r_ba = fz_norm_distance((sect_len != 0) + ti.ba_len, sect_len + sect_ba_len, c);
                    return fmax(result, fmax(r_ab, r_ba));
                };
                auto partial = [&](const uint64_t *peq, int m, const TextRef &t, double c) {
                    return fz_partial_from_best(fz_partial_best<NW, CTA_ROW>(peq, m, t), m == 0 && t.n == 0, c);
                };
                auto partial_token_ratio = [&](double c) -> double {
                    tok();
                    if (ti.n_common) return 100.0;
                    const double result = partial(peq1, las, t1, c);
                    if (na_all == na && nb_all == nb) return result;
                    c = fmax(c, result);
                    return fmax(result, partial(peq2, lau, t2, c));
                };

                double sc = 0.0;
                switch (sc_id) {
                    case FZ_RATIO: sc = fz_ratio(fz_lcs<NW>(peq0, la, t0), la, lb, cut); break;
                    case FZ_QRATIO: sc = (la == 0 || lb == 0) ? 0.0 : fz_ratio(fz_lcs<NW>(peq0, la, t0), la, lb, cut); break;
                    case FZ_PARTIAL: sc = partial(peq0, la, t0, cut); break;
                    case FZ_TSORT: sc = token_sort(cut); break;
                    case FZ_TSET: sc = token_set(cut); break;
                    case FZ_TRATIO: sc = fmax(token_set(cut), token_sort(cut)); break;
                    case FZ_PTSORT: sc = partial(peq1, las, t1, cut); break;
                    case FZ_PTSET: {
                        if (na == 0 || nb == 0) { sc = 0.0; break; }
                        tok();
                        sc = ti.n_common ? 100.0 : partial(peq2, lau, t2, cut);
                        break;
                    }
                    case FZ_PTRATIO: sc = partial_token_ratio(cut); break;
                    default: {                                  // WRatio
                        if (la == 0 || lb == 0) { sc = 0.0; break; }
                        const double len_ratio = la > lb ? __ddiv_rn((double)la, (double)lb) : __ddiv_rn((double)lb, (double)la);
                        double end_ratio = fz_ratio(fz_lcs<NW>(peq0, la, t0), la, lb, cut);
                        double c = cut;
                        if (len_ratio < 1.5) {
                            c = __ddiv_rn(fmax(c, end_ratio), 0.95);
                            sc = fmax(end_ratio, __dmul_rn(fmax(token_set(c), token_sort(c)), 0.95));
                            break;
                        }
                        const double ps = len_ratio <= 8.0 ? 0.9 : 0.6;
                        c = __ddiv_rn(fmax(c, end_ratio), ps);
                        end_ratio = fmax(end_ratio, __dmul_rn(partial(peq0, la, t0, c), ps));
                        c = __ddiv_rn(fmax(c, end_ratio), 0.95);
                        sc = fmax(end_ratio, __dmul_rn(__dmul_rn(partial_token_ratio(c), 0.95), ps));
                    }
                }
                if constexpr (TOPK) { if (sc >= P.cutoff) { cand_s = sc; cand_j = orig; } }
                else if (sc >= P.cutoff) best.offer(sc, orig);
            } while (0);
            if constexpr (TOPK) top.offer(cand_s, cand_j);
        }
        if constexpr (CTA_ROW) {
            if constexpr (TOPK) {
                if (merge_cta(top, sh_s, sh_j)) {
                    const size_t o = ((size_t)blockIdx.y * P.n_from + i) * P.k;
                    top.store(P.part_idx + o, P.part_score + o);
                }
            } else if (merge_cta(best, sh_s, sh_j)) {
                const size_t o = (size_t)blockIdx.y * P.n_from + i;
                best.store(P.part_idx + o, P.part_score + o, nullptr);
            }
            continue;                                      // (claim_row_cta's barrier ends the row)
        }
        if constexpr (TOPK) {
            const size_t o = ((size_t)blockIdx.y * P.n_from + i) * P.k;
            top.store(P.part_idx + o, P.part_score + o);
        } else {
            const size_t o = (size_t)blockIdx.y * P.n_from + i;
            best.store(P.part_idx + o, P.part_score + o, nullptr);
        }
        __syncwarp();
    }
}

template <int NW, bool TOPK>
static int launch_fuzz(const FuzzParams &P, int sms, cudaStream_t st) {
    if constexpr (NW >= 8) {
        constexpr int WARPS = 4;
        return launch_ctas(fuzz_kernel<NW, WARPS, TOPK>, WARPS, fz_cta_smem(NW, WARPS, P.scorer), P.n_ids, P.n_splits, sms, st, P);
    } else {
        constexpr int WARPS = NW == 1 ? 4 : NW == 2 ? 2 : 1;
        return launch_rows(fuzz_kernel<NW, WARPS, TOPK>, WARPS, (size_t)WARPS * 3 * 256 * NW * 8, P.n_ids, P.n_splits, sms, st, P);
    }
}

// the 38 pointers of the C ABI (order: include/pfz.h) -> FuzzParams; part_idx / part_score as the caller's entry point lays them out
template <bool TOPK>
static int run_fuzz(const void *const *ptrs, int32_t n_from, int32_t n_ids, int32_t n_words, int32_t n_to, int32_t scorer,
                    double score_cutoff, int32_t exclude_self, int64_t self_shift, int32_t n_splits, int32_t k_out, void *stream) {
    cudaStream_t st = as_stream(stream);
    FuzzParams P;
    int k = 0;
    auto side = [&](FuzzSide &S) {
        for (int v = 0; v < 3; ++v) { S.blob[v] = (const uint32_t *)ptrs[k++]; S.off[v] = (const int64_t *)ptrs[k++]; }
        S.tok_ptr = (const int32_t *)ptrs[k++]; S.tok_ids = (const int32_t *)ptrs[k++]; S.sig = (const uint64_t *)ptrs[k++];
        S.n_tok_all = (const int32_t *)ptrs[k++];
    };
    side(P.F); side(P.T);                                                           // 2 x 10
    P.from_ids = (const int32_t *)ptrs[k++]; P.sym_table = (const uint8_t *)ptrs[k++];   // 22
    for (int v = 0; v < 3; ++v) { P.packed[v] = (const uint32_t *)ptrs[k++]; P.grp_off[v] = (const int64_t *)ptrs[k++]; P.slen[v] = (const int32_t *)ptrs[k++]; }   // 31
    P.sorig = (const int32_t *)ptrs[k++]; P.tok_blob = (const uint32_t *)ptrs[k++]; P.tok_off = (const int64_t *)ptrs[k++];     // 34
    P.part_idx = (int32_t *)ptrs[k++]; P.part_score = (double *)ptrs[k++]; P.counter = (int32_t *)ptrs[k++];                  // 37
    k++;                                                                            // 38: reserved
    P.n_ids = n_ids; P.n_to = n_to; P.scorer = scorer; P.cutoff = score_cutoff; P.exclude_self = exclude_self; P.self_shift = self_shift;
    P.n_splits = n_splits; P.n_from = n_from; P.k = k_out;
    int sms = 0;
    if (start_rows(P.counter, n_splits, st, &sms)) return 1;
    if (n_words == 1) return launch_fuzz<1, TOPK>(P, sms, st);
    if (n_words == 2) return launch_fuzz<2, TOPK>(P, sms, st);
    if (n_words == 4) return launch_fuzz<4, TOPK>(P, sms, st);
    if (n_words == 8) return launch_fuzz<8, TOPK>(P, sms, st);
    return launch_fuzz<16, TOPK>(P, sms, st);
}

}  // namespace pfz

using namespace pfz;

extern "C" {

/* ptrs: 38 device pointers in the order of PfzFuzzArgs below (one flat array keeps the C ABI free of structs) */
int pfz_fuzz_argbest(const void *const *ptrs, int32_t n_ptrs, int32_t n_from, int32_t n_ids, int32_t n_words, int32_t n_to, int32_t scorer,
                     double score_cutoff, int32_t exclude_self, int64_t self_shift, int32_t n_splits, void *stream) {
    PFZ_REQUIRE(n_ptrs == 38, "pfz_fuzz_argbest: expected 38 pointers, got %d", n_ptrs);
    PFZ_REQUIRE(scorer >= FZ_RATIO && scorer <= FZ_WRATIO, "pfz_fuzz_argbest: unknown scorer %d", scorer);
    PFZ_REQUIRE(n_words == 1 || n_words == 2 || n_words == 4 || n_words == 8 || n_words == 16,
                "pfz_fuzz_argbest: n_words %d unsupported (1, 2, 4, 8, 16: from-strings up to 1024 code points)", n_words);
    PFZ_REQUIRE(n_splits >= 1, "pfz_fuzz_argbest: n_splits < 1");
    if (n_ids <= 0 || n_to <= 0) return 0;
    return run_fuzz<false>(ptrs, n_from, n_ids, n_words, n_to, scorer, score_cutoff, exclude_self, self_shift, n_splits, 1, stream);
}

/* ptrs: as pfz_fuzz_argbest, with part_idx / part_score laid out [n_splits][n_from][k] */
int pfz_fuzz_topk(const void *const *ptrs, int32_t n_ptrs, int32_t n_from, int32_t n_ids, int32_t n_words, int32_t n_to, int32_t scorer,
                  double score_cutoff, int32_t exclude_self, int64_t self_shift, int32_t n_splits, int32_t k, void *stream) {
    PFZ_REQUIRE(n_ptrs == 38, "pfz_fuzz_topk: expected 38 pointers, got %d", n_ptrs);
    PFZ_REQUIRE(scorer >= FZ_RATIO && scorer <= FZ_WRATIO, "pfz_fuzz_topk: unknown scorer %d", scorer);
    PFZ_REQUIRE(n_words == 1 || n_words == 2 || n_words == 4 || n_words == 8 || n_words == 16,
                "pfz_fuzz_topk: n_words %d unsupported (1, 2, 4, 8, 16: from-strings up to 1024 code points)", n_words);
    PFZ_REQUIRE(n_splits >= 1, "pfz_fuzz_topk: n_splits < 1");
    PFZ_REQUIRE(k >= 1 && k <= 32, "pfz_fuzz_topk: k=%d unsupported (1..32)", k);
    if (n_ids <= 0 || n_to <= 0) return 0;
    return run_fuzz<true>(ptrs, n_from, n_ids, n_words, n_to, scorer, score_cutoff, exclude_self, self_shift, n_splits, k, stream);
}
}
