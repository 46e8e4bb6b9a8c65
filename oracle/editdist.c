/* oracle/editdist.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the all-pairs edit-distance scorer that the reference delegates to the
 * third-party package `rapidfuzz` (pin: rapidfuzz>=0.13.1, reference setup.py:20; not installed and
 * not installable here -> "parity unpinned" at the package boundary; the reference's tests hold no
 * numeric vectors, only `test_score_cutoff` (tests/models/test_rapidfuzz.py:29-36)).
 * Call sites restated:
 *     polyfuzz/models/_rapidfuzz.py:99-113  process.extractOne(q, to_list, score_cutoff, scorer)
 *     polyfuzz/models/_distance.py:89-102   [scorer(q, t) for t in to_list]; np.argmax (first max)
 * Published definitions followed (rapidfuzz docs):
 *     Levenshtein, unit costs (insert/delete/substitute = 1), on Python code points
 *     Indel distance = |a| + |b| - 2*LCS(a,b)
 *     fuzz.ratio(a,b) = (1 - indel/(|a|+|b|)) * 100      (100 when both are empty)
 *     Levenshtein.normalized_similarity = 1 - d/max(|a|,|b|)   (1 when both are empty)
 *     extractOne = first choice with the maximal score among those with score >= score_cutoff
 * The DP below is the textbook Wagner-Fischer recurrence -- deliberately NOT the bit-parallel
 * algorithm the CUDA kernel uses, so that the two are independent.  A scalar Myers/Hyyro version
 * is included only as the faster CPU timing baseline (it is itself checked against the DP).
 *
 * Strings are UTF-32 code points in one blob with an offsets array (n+1 entries).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

enum { ORACLE_LEV = 0, ORACLE_INDEL = 1, ORACLE_NORM_LEV = 2, ORACLE_RATIO = 3 };

static int32_t lev_dp(const uint32_t *a, int32_t la, const uint32_t *b, int32_t lb, int32_t *row) {
    for (int32_t j = 0; j <= lb; ++j) row[j] = j;
    for (int32_t i = 1; i <= la; ++i) {
        int32_t diag = row[0];
        row[0] = i;
        for (int32_t j = 1; j <= lb; ++j) {
            int32_t up = row[j];
            int32_t best = diag + (a[i - 1] != b[j - 1]);
            if (up + 1 < best) best = up + 1;
            if (row[j - 1] + 1 < best) best = row[j - 1] + 1;
            diag = up;
            row[j] = best;
        }
    }
    return row[lb];
}

static int32_t lcs_dp(const uint32_t *a, int32_t la, const uint32_t *b, int32_t lb, int32_t *row) {
    for (int32_t j = 0; j <= lb; ++j) row[j] = 0;
    for (int32_t i = 1; i <= la; ++i) {
        int32_t diag = 0;
        for (int32_t j = 1; j <= lb; ++j) {
            int32_t up = row[j];
            int32_t best = (a[i - 1] == b[j - 1]) ? diag + 1 : (up > row[j - 1] ? up : row[j - 1]);
            diag = up;
            row[j] = best;
        }
    }
    return row[lb];
}

int32_t oracle_levenshtein(const uint32_t *a, int32_t la, const uint32_t *b, int32_t lb) {
    int32_t *row = (int32_t *)malloc(sizeof(int32_t) * (size_t)(lb + 1));
    int32_t d = lev_dp(a, la, b, lb, row);
    free(row);
    return d;
}

int32_t oracle_indel(const uint32_t *a, int32_t la, const uint32_t *b, int32_t lb) {
    int32_t *row = (int32_t *)malloc(sizeof(int32_t) * (size_t)(lb + 1));
    int32_t l = lcs_dp(a, la, b, lb, row);
    free(row);
    return la + lb - 2 * l;
}

static double score_of(int metric, int32_t d, int32_t la, int32_t lb) {
    switch (metric) {
        case ORACLE_LEV:
        case ORACLE_INDEL: return -(double)d;      /* raw distances: best = smallest */
        case ORACLE_NORM_LEV: {
            int32_t m = la > lb ? la : lb;
            return m ? 1.0 - (double)d / (double)m : 1.0;
        }
        default: { /* ORACLE_RATIO */
            int32_t m = la + lb;
            return m ? (1.0 - (double)d / (double)m) * 100.0 : 100.0;
        }
    }
}

static int32_t dist_of(int metric, const uint32_t *a, int32_t la, const uint32_t *b, int32_t lb, int32_t *row) {
    if (metric == ORACLE_LEV || metric == ORACLE_NORM_LEV) return lev_dp(a, la, b, lb, row);
    return la + lb - 2 * lcs_dp(a, la, b, lb, row);
}

static int32_t max_len(const int64_t *offs, int32_t n) {
    int32_t m = 0;
    for (int32_t i = 0; i < n; ++i) { int32_t l = (int32_t)(offs[i + 1] - offs[i]); if (l > m) m = l; }
    return m;
}

/* full distance matrix, int32 [n_from x n_to] */
int oracle_editdist_matrix(const uint32_t *fb, const int64_t *fo, int32_t n_from,
                           const uint32_t *tb, const int64_t *to, int32_t n_to,
                           int32_t metric, int32_t *dist, int32_t n_threads)
{
    int32_t ml = max_len(to, n_to);
    int nt = n_threads > 1 ? n_threads : 1;
#ifdef _OPENMP
#pragma omp parallel num_threads(nt)
#endif
    {
        int32_t *row = (int32_t *)malloc(sizeof(int32_t) * (size_t)(ml + 1));
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 4)
#endif
        for (int32_t i = 0; i < n_from; ++i) {
            const uint32_t *a = fb + fo[i]; int32_t la = (int32_t)(fo[i + 1] - fo[i]);
            for (int32_t j = 0; j < n_to; ++j) {
                const uint32_t *b = tb + to[j]; int32_t lb = (int32_t)(to[j + 1] - to[j]);
                dist[(size_t)i * n_to + j] = dist_of(metric, a, la, b, lb, row);
            }
        }
        free(row);
    }
    return 0;
}

/* RATIO's cutoff has rapidfuzz's two steps: fuzz.ratio keeps ns = 1 - d/m only if ns >= cutoff/100 and returns ns*100,
 * then extractOne keeps that score only if it is >= cutoff.  The two disagree whenever (ns*100)/100 != ns in doubles.
 * NORM_LEV (Levenshtein.normalized_similarity) has no /100 step: one test. */
static int passes_cutoff(int metric, int32_t d, int32_t la, int32_t lb, double s, double score_cutoff) {
    if (metric == ORACLE_NORM_LEV) return s >= score_cutoff;
    if (metric != ORACLE_RATIO) return 1;
    int32_t m = la + lb;
    double ns = m ? 1.0 - (double)d / (double)m : 1.0;
    return ns >= score_cutoff / 100.0 && s >= score_cutoff;
}

/* per from-row best match: first index with maximal score among the candidates that pass the cutoff
 * (metric LEV/INDEL: score = -distance, cutoff ignored).  exclude_self: skip j == i + self_shift. */
int oracle_editdist_argbest(const uint32_t *fb, const int64_t *fo, int32_t n_from,
                            const uint32_t *tb, const int64_t *to, int32_t n_to,
                            int32_t metric, double score_cutoff, int32_t exclude_self, int64_t self_shift,
                            int32_t *best_idx, double *best_score, int32_t *best_dist, int32_t n_threads)
{
    int32_t ml = max_len(to, n_to);
    int nt = n_threads > 1 ? n_threads : 1;
#ifdef _OPENMP
#pragma omp parallel num_threads(nt)
#endif
    {
        int32_t *row = (int32_t *)malloc(sizeof(int32_t) * (size_t)(ml + 1));
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 4)
#endif
        for (int32_t i = 0; i < n_from; ++i) {
            const uint32_t *a = fb + fo[i]; int32_t la = (int32_t)(fo[i + 1] - fo[i]);
            int32_t bi = -1, bd = -1; double bs = 0.0;
            for (int32_t j = 0; j < n_to; ++j) {
                if (exclude_self && (int64_t)j == (int64_t)i + self_shift) continue;
                const uint32_t *b = tb + to[j]; int32_t lb = (int32_t)(to[j + 1] - to[j]);
                int32_t d = dist_of(metric, a, la, b, lb, row);
                double s = score_of(metric, d, la, lb);
                if (!passes_cutoff(metric, d, la, lb, s, score_cutoff)) continue;
                if (bi < 0 || s > bs) { bi = j; bs = s; bd = d; }
            }
            best_idx[i] = bi; best_score[i] = bi < 0 ? 0.0 : bs; best_dist[i] = bd;
        }
        free(row);
    }
    return 0;
}

/* ---- scalar 64-bit Myers (1999) / Hyyro (2003) -- CPU TIMING BASELINE ONLY ------------------
 * Pattern (from-string) must be <= 64 code points and every code point < 65536 for the direct
 * Peq table; otherwise falls back to the DP above.  Checked against the DP in tests. */
static int32_t myers64(const uint64_t *peq_lo /*[256]*/, const uint32_t *pat, int32_t m,
                       const uint32_t *txt, int32_t n) {
    if (m == 0) return n;
    uint64_t Pv = ~0ULL, Mv = 0; int32_t score = m; uint64_t top = 1ULL << (m - 1);
    for (int32_t j = 0; j < n; ++j) {
        uint32_t c = txt[j];
        uint64_t Eq = 0;
        if (c < 256) Eq = peq_lo[c];
        else { for (int32_t i = 0; i < m; ++i) if (pat[i] == c) Eq |= 1ULL << i; }
        uint64_t Xv = Eq | Mv;
        uint64_t Xh = (((Eq & Pv) + Pv) ^ Pv) | Eq;
        uint64_t Ph = Mv | ~(Xh | Pv);
        uint64_t Mh = Pv & Xh;
        if (Ph & top) ++score;
        if (Mh & top) --score;
        Ph = (Ph << 1) | 1ULL; Mh <<= 1;
        Pv = Mh | ~(Xv | Ph);
        Mv = Ph & Xv;
    }
    return score;
}

int oracle_lev_argbest_myers(const uint32_t *fb, const int64_t *fo, int32_t n_from,
                             const uint32_t *tb, const int64_t *to, int32_t n_to,
                             int32_t *best_idx, double *best_score, int32_t *best_dist, int32_t n_threads)
{
    int32_t ml = max_len(to, n_to);
    int nt = n_threads > 1 ? n_threads : 1;
#ifdef _OPENMP
#pragma omp parallel num_threads(nt)
#endif
    {
        int32_t *row = (int32_t *)malloc(sizeof(int32_t) * (size_t)(ml + 1));
        uint64_t peq[256];
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 4)
#endif
        for (int32_t i = 0; i < n_from; ++i) {
            const uint32_t *a = fb + fo[i]; int32_t la = (int32_t)(fo[i + 1] - fo[i]);
            int use_bp = la <= 64;
            if (use_bp) {
                memset(peq, 0, sizeof(peq));
                for (int32_t p = 0; p < la; ++p) if (a[p] < 256) peq[a[p]] |= 1ULL << p;
            }
            int32_t bi = -1, bd = -1; double bs = 0.0;
            for (int32_t j = 0; j < n_to; ++j) {
                const uint32_t *b = tb + to[j]; int32_t lb = (int32_t)(to[j + 1] - to[j]);
                int32_t d = use_bp ? myers64(peq, a, la, b, lb) : lev_dp(a, la, b, lb, row);
                int32_t m = la > lb ? la : lb;
                double s = m ? 1.0 - (double)d / (double)m : 1.0;
                if (bi < 0 || s > bs) { bi = j; bs = s; bd = d; }
            }
            best_idx[i] = bi; best_score[i] = bi < 0 ? 0.0 : bs; best_dist[i] = bd;
        }
        free(row);
    }
    return 0;
}
