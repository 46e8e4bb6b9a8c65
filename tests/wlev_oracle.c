/* tests/wlev_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of weighted Levenshtein (rapidfuzz.distance.Levenshtein with weights = (insertion, deletion, substitution))
 * on Python code points, the oracle of K3's wlev_kernel:
 *     D(a, b) = the textbook Wagner-Fischer minimum, in int64:
 *               d[i][0] = i * wd, d[0][j] = j * wi,
 *               d[i][j] = min(d[i-1][j] + wd, d[i][j-1] + wi, d[i-1][j-1] + (a[i-1] == b[j-1] ? 0 : ws))
 *     M(a, b) = min(m*wd + n*wi, n*ws + (m-n)*wd) when m >= n, else min(m*wd + n*wi, m*ws + (n-m)*wi)   (m = |a|, n = |b|)
 *     score   = 1 - D/M in IEEE double (1 when M == 0)
 *     top-k   = per from-row the k best to-indices with score >= score_cutoff, key score desc then index asc; exclude_self
 *               skips j == i + self_shift.  Empty slots are (-1, 0.0, -1).
 * Deliberately the full three-way minimum over two int64 rows, walked row by row over the from-string, not the kernel's
 * unconditional-diagonal, column-relative int32 recurrence streamed over the to-string.
 * Strings are UTF-32 code points in one blob with an offsets array (n+1 entries).
 */
#include <stdint.h>
#include <stdlib.h>
#ifdef _OPENMP
#include <omp.h>
#endif

static int64_t wlev_dp(const uint32_t *a, int32_t la, const uint32_t *b, int32_t lb, int64_t wi, int64_t wd, int64_t ws,
                       int64_t *prev, int64_t *cur) {
    for (int32_t j = 0; j <= lb; ++j) prev[j] = (int64_t)j * wi;
    for (int32_t i = 1; i <= la; ++i) {
        cur[0] = (int64_t)i * wd;
        for (int32_t j = 1; j <= lb; ++j) {
            int64_t best = prev[j - 1] + (a[i - 1] == b[j - 1] ? 0 : ws);
            if (prev[j] + wd < best) best = prev[j] + wd;
            if (cur[j - 1] + wi < best) best = cur[j - 1] + wi;
            cur[j] = best;
        }
        int64_t *t = prev; prev = cur; cur = t;
    }
    return prev[lb];
}

static int64_t wlev_max(int64_t m, int64_t n, int64_t wi, int64_t wd, int64_t ws) {
    const int64_t del_ins = m * wd + n * wi;
    const int64_t other = m >= n ? n * ws + (m - n) * wd : m * ws + (n - m) * wi;
    return other < del_ins ? other : del_ins;
}

static int32_t max_len(const int64_t *offs, int32_t n) {
    int32_t m = 0;
    for (int32_t i = 0; i < n; ++i) { int32_t l = (int32_t)(offs[i + 1] - offs[i]); if (l > m) m = l; }
    return m;
}

/* D and M matrices, int64 [n_from x n_to] */
int oracle_wlev_matrix(const uint32_t *fb, const int64_t *fo, int32_t n_from, const uint32_t *tb, const int64_t *to, int32_t n_to,
                       int32_t wi, int32_t wd, int32_t ws, int64_t *dist, int64_t *maxm, int32_t n_threads) {
    const size_t cols = (size_t)max_len(to, n_to) + 1;
    int nt = n_threads > 1 ? n_threads : 1;
    (void)nt;
#ifdef _OPENMP
#pragma omp parallel num_threads(nt)
#endif
    {
        int64_t *buf = (int64_t *)malloc(sizeof(int64_t) * 2 * cols);
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 4)
#endif
        for (int32_t i = 0; i < n_from; ++i) {
            const uint32_t *a = fb + fo[i]; int32_t la = (int32_t)(fo[i + 1] - fo[i]);
            for (int32_t j = 0; j < n_to; ++j) {
                const int32_t lb = (int32_t)(to[j + 1] - to[j]);
                dist[(size_t)i * n_to + j] = wlev_dp(a, la, tb + to[j], lb, wi, wd, ws, buf, buf + cols);
                maxm[(size_t)i * n_to + j] = wlev_max(la, lb, wi, wd, ws);
            }
        }
        free(buf);
    }
    return 0;
}

/* per from-row the k best under the canonical key: idx int32 / score double / dist int64 [n_from x k] */
int oracle_wlev_topk(const uint32_t *fb, const int64_t *fo, int32_t n_from, const uint32_t *tb, const int64_t *to, int32_t n_to,
                     int32_t wi, int32_t wd, int32_t ws, int32_t k, double score_cutoff, int32_t exclude_self, int64_t self_shift,
                     int32_t *idx, double *score, int64_t *dist, int32_t n_threads) {
    const size_t cols = (size_t)max_len(to, n_to) + 1;
    int nt = n_threads > 1 ? n_threads : 1;
    (void)nt;
#ifdef _OPENMP
#pragma omp parallel num_threads(nt)
#endif
    {
        int64_t *buf = (int64_t *)malloc(sizeof(int64_t) * 2 * cols);
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 4)
#endif
        for (int32_t i = 0; i < n_from; ++i) {
            const uint32_t *a = fb + fo[i]; int32_t la = (int32_t)(fo[i + 1] - fo[i]);
            int32_t *ri = idx + (size_t)i * k; double *rs = score + (size_t)i * k; int64_t *rd = dist + (size_t)i * k;
            int32_t cnt = 0;
            for (int32_t j = 0; j < n_to; ++j) {
                if (exclude_self && (int64_t)j == (int64_t)i + self_shift) continue;
                const int32_t lb = (int32_t)(to[j + 1] - to[j]);
                const int64_t d = wlev_dp(a, la, tb + to[j], lb, wi, wd, ws, buf, buf + cols);
                const int64_t mx = wlev_max(la, lb, wi, wd, ws);
                const double s = mx ? 1.0 - (double)d / (double)mx : 1.0;
                if (!(s >= score_cutoff)) continue;
                /* j ascends, so among equal scores the earlier entry stays first: insert after every score >= s */
                int32_t pos = cnt;
                while (pos > 0 && rs[pos - 1] < s) --pos;
                if (pos >= k) continue;
                const int32_t last = cnt < k ? cnt : k - 1;
                for (int32_t q = last; q > pos; --q) { ri[q] = ri[q - 1]; rs[q] = rs[q - 1]; rd[q] = rd[q - 1]; }
                ri[pos] = j; rs[pos] = s; rd[pos] = d;
                if (cnt < k) ++cnt;
            }
            for (int32_t q = cnt; q < k; ++q) { ri[q] = -1; rs[q] = 0.0; rd[q] = -1; }
        }
        free(buf);
    }
    return 0;
}
