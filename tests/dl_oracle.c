/* tests/dl_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of unrestricted Damerau-Levenshtein (rapidfuzz.distance.DamerauLevenshtein, jellyfish's
 * damerau_levenshtein_distance) on Python code points, the oracle of K3's dl_kernel:
 *     dl(a, b) = the fewest insertions, deletions, substitutions and swaps of two adjacent characters, where a swapped pair
 *                may be edited again (dl("CA", "ABC") = 2).  DP: Lowrance & Wagner (1975) with unit costs, the textbook
 *                full (la + 2) x (lb + 2) matrix and a code point -> last row map:
 *                d[i][j] = min(d[i-1][j-1] + (a[i-1] != b[j-1]), d[i][j-1] + 1, d[i-1][j] + 1,
 *                              d[k-1][l-1] + (i - k - 1) + 1 + (j - l - 1)),
 *                k = last row < i with a[k-1] == b[j-1], l = last column < j with b[l-1] == a[i-1]
 *     DamerauLevenshtein.normalized_similarity = 1 - dl / max(|a|, |b|)   (1 when both are empty)
 *     best match = first to-index with the maximal score among score >= score_cutoff (normalized); for the raw distance,
 *                  score = -distance and no cutoff.  exclude_self skips j == i + self_shift.
 * Deliberately not the column-streamed linear-space formulation the CUDA kernel uses.
 * Strings are UTF-32 code points in one blob with an offsets array (n+1 entries).
 */
#include <stdint.h>
#include <stdlib.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define N_CP 0x110000

/* d: (la + 2) x (lb + 2) work matrix, row-major with stride lb + 2; da: last row of each code point (all 0 on entry and exit) */
static int32_t dl_dp(const uint32_t *a, int32_t la, const uint32_t *b, int32_t lb, int32_t *d, int32_t *da) {
    const int32_t W = lb + 2, INF = la + lb;
#define D(i, j) d[(size_t)(i) * W + (j)]
    D(0, 0) = INF;
    for (int32_t i = 0; i <= la; ++i) { D(i + 1, 0) = INF; D(i + 1, 1) = i; }
    for (int32_t j = 0; j <= lb; ++j) { D(0, j + 1) = INF; D(1, j + 1) = j; }
    for (int32_t i = 1; i <= la; ++i) {
        int32_t db = 0;
        for (int32_t j = 1; j <= lb; ++j) {
            const int32_t k = b[j - 1] < N_CP ? da[b[j - 1]] : 0, l = db;
            int32_t cost = 1;
            if (a[i - 1] == b[j - 1]) { cost = 0; db = j; }
            int32_t best = D(i, j) + cost;
            if (D(i + 1, j) + 1 < best) best = D(i + 1, j) + 1;
            if (D(i, j + 1) + 1 < best) best = D(i, j + 1) + 1;
            const int32_t tr = D(k, l) + (i - k - 1) + 1 + (j - l - 1);
            if (tr < best) best = tr;
            D(i + 1, j + 1) = best;
        }
        if (a[i - 1] < N_CP) da[a[i - 1]] = i;
    }
    const int32_t r = D(la + 1, lb + 1);
    for (int32_t i = 0; i < la; ++i) if (a[i] < N_CP) da[a[i]] = 0;
#undef D
    return r;
}

static int32_t max_len(const int64_t *offs, int32_t n) {
    int32_t m = 0;
    for (int32_t i = 0; i < n; ++i) { int32_t l = (int32_t)(offs[i + 1] - offs[i]); if (l > m) m = l; }
    return m;
}

/* full DL distance matrix, int32 [n_from x n_to] */
int oracle_dl_matrix(const uint32_t *fb, const int64_t *fo, int32_t n_from, const uint32_t *tb, const int64_t *to, int32_t n_to,
                     int32_t *dist, int32_t n_threads) {
    const size_t cells = (size_t)(max_len(fo, n_from) + 2) * (size_t)(max_len(to, n_to) + 2);
    int nt = n_threads > 1 ? n_threads : 1;
    (void)nt;
#ifdef _OPENMP
#pragma omp parallel num_threads(nt)
#endif
    {
        int32_t *d = (int32_t *)malloc(sizeof(int32_t) * cells);
        int32_t *da = (int32_t *)calloc(N_CP, sizeof(int32_t));
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 4)
#endif
        for (int32_t i = 0; i < n_from; ++i) {
            const uint32_t *a = fb + fo[i]; int32_t la = (int32_t)(fo[i + 1] - fo[i]);
            for (int32_t j = 0; j < n_to; ++j)
                dist[(size_t)i * n_to + j] = dl_dp(a, la, tb + to[j], (int32_t)(to[j + 1] - to[j]), d, da);
        }
        free(d); free(da);
    }
    return 0;
}

/* per from-row best match (normalized = 1: norm_dl with score_cutoff; 0: raw distance, score = -distance, no cutoff) */
int oracle_dl_argbest(const uint32_t *fb, const int64_t *fo, int32_t n_from, const uint32_t *tb, const int64_t *to, int32_t n_to,
                      int32_t normalized, double score_cutoff, int32_t exclude_self, int64_t self_shift,
                      int32_t *best_idx, double *best_score, int32_t *best_dist, int32_t n_threads) {
    const size_t cells = (size_t)(max_len(fo, n_from) + 2) * (size_t)(max_len(to, n_to) + 2);
    int nt = n_threads > 1 ? n_threads : 1;
    (void)nt;
#ifdef _OPENMP
#pragma omp parallel num_threads(nt)
#endif
    {
        int32_t *d = (int32_t *)malloc(sizeof(int32_t) * cells);
        int32_t *da = (int32_t *)calloc(N_CP, sizeof(int32_t));
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 4)
#endif
        for (int32_t i = 0; i < n_from; ++i) {
            const uint32_t *a = fb + fo[i]; int32_t la = (int32_t)(fo[i + 1] - fo[i]);
            int32_t bi = -1, bd = -1; double bs = 0.0;
            for (int32_t j = 0; j < n_to; ++j) {
                if (exclude_self && (int64_t)j == (int64_t)i + self_shift) continue;
                int32_t lb = (int32_t)(to[j + 1] - to[j]);
                int32_t dd = dl_dp(a, la, tb + to[j], lb, d, da);
                double s;
                if (normalized) {
                    int32_t m = la > lb ? la : lb;
                    s = m ? 1.0 - (double)dd / (double)m : 1.0;
                    if (!(s >= score_cutoff)) continue;
                } else {
                    s = -(double)dd;                /* raw distance: best = smallest */
                }
                if (bi < 0 || s > bs) { bi = j; bs = s; bd = dd; }
            }
            best_idx[i] = bi; best_score[i] = bi < 0 ? 0.0 : bs; best_dist[i] = bd;
        }
        free(d); free(da);
    }
    return 0;
}
