"""Plain-Python restatement of rapidfuzz 3.x's Indel, LCSseq, Hamming, Prefix and Postfix normalised similarities (TEST
INFRASTRUCTURE, NOT PRODUCT CODE), written from their definitions on code points, s1 = the from-string (length m), s2 = the
to-string (length n), processor=None:

    metric          distance d                                        maximum M
    norm_indel      m + n - 2 LCS                                     m + n
    norm_lcsseq     M - LCS                                           max(m, n)
    norm_hamming    mismatches at positions < min(m, n) + |m - n|     max(m, n)     (pad=True, rapidfuzz 3's default)
    norm_prefix     M - the common prefix length                      max(m, n)
    norm_postfix    M - the common suffix length                      max(m, n)

and the normalised similarity 1.0 - float(d) / float(M), 1.0 when M = 0.  LCS is the textbook O(m n) dynamic programme;
lcs_matrix can take tests/lcs_oracle.c's C transcription of the same programme for long strings.  Nothing here shares a
formulation with the kernels."""
import numpy as np

METRICS = ("norm_indel", "norm_lcsseq", "norm_hamming", "norm_prefix", "norm_postfix")


def lcs_len(a, b):
    """Length of the longest common subsequence of a and b (textbook DP, one row)."""
    if not a or not b:
        return 0
    prev = [0] * (len(b) + 1)
    for ca in a:
        cur = [0]
        for j, cb in enumerate(b, 1):
            cur.append(prev[j - 1] + 1 if ca == cb else max(prev[j], cur[j - 1]))
        prev = cur
    return prev[-1]


def hamming_mismatches(a, b):
    """Positions < min(|a|, |b|) where a and b differ."""
    return sum(1 for x, y in zip(a, b) if x != y)


def common_prefix(a, b):
    k = 0
    for x, y in zip(a, b):
        if x != y:
            break
        k += 1
    return k


def common_suffix(a, b):
    return common_prefix(a[::-1], b[::-1])


def normalized(d, mx):
    """rapidfuzz's normalized_similarity from the distance and the maximum: 1 - d/M in float64, 1.0 when M = 0."""
    return 1.0 - float(d) / float(mx) if mx else 1.0


def dist_max(metric, a, b, lcs=None):
    """(d, M) of one pair; lcs: the pair's LCS length when known (Indel / LCSseq)."""
    m, n = len(a), len(b)
    if metric in ("norm_indel", "norm_lcsseq"):
        c = lcs_len(a, b) if lcs is None else lcs
        if metric == "norm_indel":
            return m + n - 2 * c, m + n
        return max(m, n) - c, max(m, n)
    if metric == "norm_hamming":
        return hamming_mismatches(a, b) + abs(m - n), max(m, n)
    if metric == "norm_prefix":
        return max(m, n) - common_prefix(a, b), max(m, n)
    if metric == "norm_postfix":
        return max(m, n) - common_suffix(a, b), max(m, n)
    raise ValueError(metric)


def similarity(metric, a, b):
    return normalized(*dist_max(metric, a, b))


def lcs_matrix(from_list, to_list, fast=True):
    """int64 [n_from, n_to] of LCS lengths: tests/lcs_oracle.c when fast, else lcs_len."""
    out = np.zeros((len(from_list), len(to_list)), dtype=np.int64)
    if fast:
        import lcs_oracle
        f = lcs_oracle.lib().oracle_lcs
        tu = [lcs_oracle._u32(t) for t in to_list]
        for i, a in enumerate(from_list):
            if not a:
                continue
            x = lcs_oracle._u32(a)
            for j, y in enumerate(tu):
                if len(y):
                    out[i, j] = f(x.ctypes.data, len(x), y.ctypes.data, len(y))
    else:
        for i, a in enumerate(from_list):
            for j, b in enumerate(to_list):
                out[i, j] = lcs_len(a, b)
    return out


def matrices(metric, from_list, to_list, lcs=None):
    """(D int64, M int64, S float64) [n_from, n_to]: distances, maxima and scores; lcs: lcs_matrix(from_list, to_list) when
    already known (Indel / LCSseq)."""
    nf, nt = len(from_list), len(to_list)
    if metric in ("norm_indel", "norm_lcsseq") and lcs is None:
        lcs = lcs_matrix(from_list, to_list)
    D = np.zeros((nf, nt), dtype=np.int64)
    M = np.zeros((nf, nt), dtype=np.int64)
    S = np.zeros((nf, nt), dtype=np.float64)
    for i, a in enumerate(from_list):
        for j, b in enumerate(to_list):
            d, mx = dist_max(metric, a, b, None if lcs is None else int(lcs[i, j]))
            D[i, j], M[i, j], S[i, j] = d, mx, normalized(d, mx)
    return D, M, S


def topk_from(S, D, k, score_cutoff=0.0, exclude_self=False, self_shift=0, allowed=None):
    """Per row the k best columns (score desc, index asc) with S >= score_cutoff, skipping column i + self_shift when
    exclude_self and, when given, columns outside allowed[i]: (idx int32 [n, k], score float64 [n, k], dist int64 [n, k]), empty
    slots (-1, 0.0, -1)."""
    n, nt = S.shape
    idx = np.full((n, k), -1, dtype=np.int32)
    sc = np.zeros((n, k), dtype=np.float64)
    dist = np.full((n, k), -1, dtype=np.int64)
    for i in range(n):
        js = np.arange(nt) if allowed is None else np.array(sorted(j for j in allowed[i] if j >= 0), dtype=np.int64)
        if len(js):
            js = js[S[i, js] >= score_cutoff]
        if exclude_self:
            js = js[js != i + self_shift]
        js = js[np.lexsort((js, -S[i, js]))][:k] if len(js) else js
        idx[i, :len(js)] = js
        sc[i, :len(js)] = S[i, js]
        dist[i, :len(js)] = D[i, js]
    return idx, sc, dist


def topk(metric, from_list, to_list, k, score_cutoff=0.0, exclude_self=False, self_shift=0):
    D, _, S = matrices(metric, from_list, to_list)
    return topk_from(S, D, k, score_cutoff, exclude_self, self_shift)


def argbest(metric, from_list, to_list, score_cutoff=0.0, exclude_self=False, self_shift=0):
    """topk with k = 1, as [n] arrays."""
    i, s, d = topk(metric, from_list, to_list, 1, score_cutoff, exclude_self, self_shift)
    return i[:, 0], s[:, 0], d[:, 0]
