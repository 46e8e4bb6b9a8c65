/* tests/jaro_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of jellyfish's jaro_similarity / jaro_winkler_similarity (long_tolerance=False, what a
 * bare function passed as EditDistance's scorer uses), called by the reference as scorer(from_string, to_string)
 * (polyfuzz/models/_distance.py:98).  Strings are UTF-32 code points.  s1 = from-string, s2 = to-string:
 *   1. l1 == 0 or l2 == 0 -> 0.0
 *   2. R = max(0, max(l1, l2) / 2 - 1)
 *   3. for i in order, s1[i] matches the LOWEST unflagged j with |i - j| <= R and s2[j] == s1[i]; m = matches
 *      (m == 0 -> 0.0)
 *   4. t = (pairs k-th flagged s1 position / k-th flagged s2 position with different characters) / 2
 *   5. jaro = (m/l1 + m/l2 + (m - t)/m) / 3            (float64, in this order)
 *   6. jaro > 0.7: p = common prefix capped at min(l1, l2, 4); p > 0 -> jw = jaro + (p*0.1) * (1.0 - jaro)
 * This is the s1-driven O(l1 * R) loop of the definition -- deliberately NOT the text-driven bit-parallel
 * formulation the CUDA kernel uses, so that the two are independent.  Build with -ffp-contract=off.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* flags: >= la + lb bytes of scratch.  *matches receives m. */
static double jaro_core(const uint32_t *a, int32_t la, const uint32_t *b, int32_t lb, int32_t winkler, int32_t *matches,
                        uint8_t *flags) {
    *matches = 0;
    if (la == 0 || lb == 0) return 0.0;
    int32_t R = (la > lb ? la : lb) / 2 - 1;
    if (R < 0) R = 0;
    uint8_t *f1 = flags, *f2 = flags + la;
    memset(flags, 0, (size_t)la + (size_t)lb);
    int32_t m = 0;
    for (int32_t i = 0; i < la; ++i) {
        const int32_t lo = i - R > 0 ? i - R : 0;
        const int32_t hi = i + R < lb - 1 ? i + R : lb - 1;
        for (int32_t j = lo; j <= hi; ++j) {
            if (!f2[j] && b[j] == a[i]) { f1[i] = f2[j] = 1; ++m; break; }
        }
    }
    *matches = m;
    if (m == 0) return 0.0;
    int32_t k = 0, trans = 0;
    for (int32_t i = 0; i < la; ++i) {
        if (!f1[i]) continue;
        while (!f2[k]) ++k;
        if (a[i] != b[k]) ++trans;
        ++k;
    }
    const int32_t t = trans / 2;
    const double dm = (double)m;
    double jaro = (dm / (double)la + dm / (double)lb + (dm - (double)t) / dm) / 3.0;
    if (winkler && jaro > 0.7) {
        int32_t cap = la < lb ? la : lb;
        if (cap > 4) cap = 4;
        int32_t p = 0;
        while (p < cap && a[p] == b[p]) ++p;
        if (p > 0) jaro = jaro + ((double)p * 0.1) * (1.0 - jaro);
    }
    return jaro;
}

double oracle_jaro_pair(const uint32_t *a, int32_t la, const uint32_t *b, int32_t lb, int32_t winkler, int32_t *matches) {
    uint8_t *flags = (uint8_t *)malloc((size_t)la + (size_t)lb + 1);
    const double s = jaro_core(a, la, b, lb, winkler, matches, flags);
    free(flags);
    return s;
}

static int32_t max_len(const int64_t *offs, int32_t n) {
    int32_t m = 0;
    for (int32_t i = 0; i < n; ++i) { int32_t l = (int32_t)(offs[i + 1] - offs[i]); if (l > m) m = l; }
    return m;
}

/* per from-row best match: first to-index with the maximal score among score >= score_cutoff;
 * exclude_self: skip j == i + self_shift.  best_dist receives the match count m of the best pair (-1 = none). */
int oracle_jaro_argbest(const uint32_t *fb, const int64_t *fo, int32_t n_from, const uint32_t *tb, const int64_t *to, int32_t n_to,
                        int32_t winkler, double score_cutoff, int32_t exclude_self, int64_t self_shift, int32_t *best_idx,
                        double *best_score, int32_t *best_dist, int32_t n_threads) {
    const size_t scratch = (size_t)max_len(fo, n_from) + (size_t)max_len(to, n_to) + 1;
    int nt = n_threads > 1 ? n_threads : 1;
#ifdef _OPENMP
#pragma omp parallel num_threads(nt)
#endif
    {
        uint8_t *flags = (uint8_t *)malloc(scratch);
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 4)
#endif
        for (int32_t i = 0; i < n_from; ++i) {
            const uint32_t *a = fb + fo[i]; int32_t la = (int32_t)(fo[i + 1] - fo[i]);
            int32_t bi = -1, bd = -1; double bs = 0.0;
            for (int32_t j = 0; j < n_to; ++j) {
                if (exclude_self && (int64_t)j == (int64_t)i + self_shift) continue;
                const uint32_t *b = tb + to[j]; int32_t lb = (int32_t)(to[j + 1] - to[j]);
                int32_t m;
                const double s = jaro_core(a, la, b, lb, winkler, &m, flags);
                if (!(s >= score_cutoff)) continue;
                if (bi < 0 || s > bs) { bi = j; bs = s; bd = m; }
            }
            best_idx[i] = bi; best_score[i] = bi < 0 ? 0.0 : bs; best_dist[i] = bd;
        }
        free(flags);
    }
    return 0;
}
