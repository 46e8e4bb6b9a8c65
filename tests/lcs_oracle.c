/* lcs_oracle.c -- textbook longest-common-subsequence length of two UTF-32 strings (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
 *
 * The O(|a| |b|) dynamic programme with one row, the same recurrence as oracle/fuzz.py's lcs_len, in C so that the
 * oracle can score strings of a few thousand code points (partial_ratio runs one LCS per window).  Deliberately not
 * bit-parallel: it shares no formulation with the kernels it checks.
 */
#include <stdint.h>
#include <stdlib.h>

int64_t oracle_lcs(const uint32_t *a, int64_t la, const uint32_t *b, int64_t lb) {
    if (la == 0 || lb == 0) return 0;
    int64_t *prev = (int64_t *)calloc((size_t)lb + 1, sizeof(int64_t));
    int64_t *cur = (int64_t *)calloc((size_t)lb + 1, sizeof(int64_t));
    if (!prev || !cur) { free(prev); free(cur); return -1; }
    for (int64_t i = 0; i < la; ++i) {
        cur[0] = 0;
        for (int64_t j = 1; j <= lb; ++j) {
            if (a[i] == b[j - 1]) cur[j] = prev[j - 1] + 1;
            else cur[j] = prev[j] >= cur[j - 1] ? prev[j] : cur[j - 1];
        }
        int64_t *t = prev; prev = cur; cur = t;
    }
    const int64_t r = prev[lb];
    free(prev); free(cur);
    return r;
}
