/* tests/osa_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of rapidfuzz.distance.OSA (optimal string alignment, also called restricted Damerau-Levenshtein) on
 * Python code points, the oracle of K3's OSA mode:
 *     osa(a, b) = the fewest insertions, deletions, substitutions and swaps of two adjacent characters, no substring
 *                 edited more than once.  DP: Wagner-Fischer plus
 *                 d[i][j] = min(d[i][j], d[i-2][j-2] + 1) when a[i-1] == b[j-2] and a[i-2] == b[j-1]
 *     OSA.normalized_similarity = 1 - osa / max(|a|, |b|)   (1 when both are empty)
 *     best match = first to-index with the maximal score among score >= score_cutoff (normalized); for the raw distance,
 *                  score = -distance and no cutoff.  exclude_self skips j == i + self_shift.
 * The DP is the textbook recurrence -- deliberately NOT the bit-parallel one the CUDA kernel uses.
 * Strings are UTF-32 code points in one blob with an offsets array (n+1 entries).
 */
#include <stdint.h>
#include <stdlib.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* three rows (work holds 3 * (lb + 1) entries): pp = row i-2, p = row i-1, c = row i */
static int32_t osa_dp(const uint32_t *a, int32_t la, const uint32_t *b, int32_t lb, int32_t *work) {
    int32_t *pp = work, *p = work + (lb + 1), *c = work + 2 * (lb + 1);
    for (int32_t j = 0; j <= lb; ++j) p[j] = j;
    for (int32_t i = 1; i <= la; ++i) {
        c[0] = i;
        for (int32_t j = 1; j <= lb; ++j) {
            int32_t best = p[j - 1] + (a[i - 1] != b[j - 1]);
            if (p[j] + 1 < best) best = p[j] + 1;
            if (c[j - 1] + 1 < best) best = c[j - 1] + 1;
            if (i > 1 && j > 1 && a[i - 1] == b[j - 2] && a[i - 2] == b[j - 1] && pp[j - 2] + 1 < best) best = pp[j - 2] + 1;
            c[j] = best;
        }
        int32_t *t = pp; pp = p; p = c; c = t;
    }
    return p[lb];
}

static int32_t max_len(const int64_t *offs, int32_t n) {
    int32_t m = 0;
    for (int32_t i = 0; i < n; ++i) { int32_t l = (int32_t)(offs[i + 1] - offs[i]); if (l > m) m = l; }
    return m;
}

/* full OSA distance matrix, int32 [n_from x n_to] */
int oracle_osa_matrix(const uint32_t *fb, const int64_t *fo, int32_t n_from, const uint32_t *tb, const int64_t *to, int32_t n_to,
                      int32_t *dist, int32_t n_threads) {
    int32_t ml = max_len(to, n_to);
    int nt = n_threads > 1 ? n_threads : 1;
    (void)nt;
#ifdef _OPENMP
#pragma omp parallel num_threads(nt)
#endif
    {
        int32_t *work = (int32_t *)malloc(sizeof(int32_t) * 3 * (size_t)(ml + 1));
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 4)
#endif
        for (int32_t i = 0; i < n_from; ++i) {
            const uint32_t *a = fb + fo[i]; int32_t la = (int32_t)(fo[i + 1] - fo[i]);
            for (int32_t j = 0; j < n_to; ++j)
                dist[(size_t)i * n_to + j] = osa_dp(a, la, tb + to[j], (int32_t)(to[j + 1] - to[j]), work);
        }
        free(work);
    }
    return 0;
}

/* per from-row best match (normalized = 1: norm_osa with score_cutoff; 0: raw distance, score = -distance, no cutoff) */
int oracle_osa_argbest(const uint32_t *fb, const int64_t *fo, int32_t n_from, const uint32_t *tb, const int64_t *to, int32_t n_to,
                       int32_t normalized, double score_cutoff, int32_t exclude_self, int64_t self_shift,
                       int32_t *best_idx, double *best_score, int32_t *best_dist, int32_t n_threads) {
    int32_t ml = max_len(to, n_to);
    int nt = n_threads > 1 ? n_threads : 1;
    (void)nt;
#ifdef _OPENMP
#pragma omp parallel num_threads(nt)
#endif
    {
        int32_t *work = (int32_t *)malloc(sizeof(int32_t) * 3 * (size_t)(ml + 1));
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 4)
#endif
        for (int32_t i = 0; i < n_from; ++i) {
            const uint32_t *a = fb + fo[i]; int32_t la = (int32_t)(fo[i + 1] - fo[i]);
            int32_t bi = -1, bd = -1; double bs = 0.0;
            for (int32_t j = 0; j < n_to; ++j) {
                if (exclude_self && (int64_t)j == (int64_t)i + self_shift) continue;
                int32_t lb = (int32_t)(to[j + 1] - to[j]);
                int32_t d = osa_dp(a, la, tb + to[j], lb, work);
                double s;
                if (normalized) {
                    int32_t m = la > lb ? la : lb;
                    s = m ? 1.0 - (double)d / (double)m : 1.0;
                    if (!(s >= score_cutoff)) continue;
                } else {
                    s = -(double)d;                 /* raw distance: best = smallest */
                }
                if (bi < 0 || s > bs) { bi = j; bs = s; bd = d; }
            }
            best_idx[i] = bi; best_score[i] = bi < 0 ? 0.0 : bs; best_dist[i] = bd;
        }
        free(work);
    }
    return 0;
}
