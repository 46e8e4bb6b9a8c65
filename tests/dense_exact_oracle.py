"""CPU oracle of the Embeddings exact mode (precision="fp64"): the canonical fp64 cosine top-k of DESIGN.md section 2.

    dot(a, b): 32 partial sums p[l] = sum over ascending t of a[32t+l] * b[32t+l] (each product rounded, then added; no
               FMA; from +0), then p[l] <- p[l] + p[l xor o] for o = 16, 8, 4, 2, 1; the result is p[0].
    x~ = x / sqrt(dot(x, x)), correctly rounded; a row with dot(x, x) == 0 stays as it is.
    score(i, j) = dot(x~_i, y~_j); candidate iff score > thr (strict) and j != i in a self-match;
    ranking (score desc, index asc); empty slots (-1, 0.0).

numpy evaluates `p + a * b` as two separately rounded operations, which is the definition."""
import numpy as np

_XOR = [np.arange(32) ^ o for o in (16, 8, 4, 2, 1)]


def _pad32(a):
    a = np.asarray(a, dtype=np.float64)
    d = a.shape[-1]
    dp = max(32, (d + 31) // 32 * 32)
    if dp == d:
        return a
    out = np.zeros(a.shape[:-1] + (dp,), dtype=np.float64)
    out[..., :d] = a
    return out


def _butterfly(p):
    for ix in _XOR:
        p = p + p[..., ix]
    return p[..., 0]


def _by_term(B):
    """B [m, d] -> [T, m, 32] (term-major, contiguous): the layout canon_dot walks."""
    B = _pad32(B)
    return np.ascontiguousarray(B.reshape(B.shape[0], -1, 32).transpose(1, 0, 2))


def canon_dot(a, B, B_by_term=None):
    """Canonical dot of a [..., d] with every row of B [m, d] -> [..., m]."""
    a = _pad32(a)
    Bt = _by_term(B) if B_by_term is None else B_by_term
    p = np.zeros(a.shape[:-1] + Bt.shape[1:], dtype=np.float64)
    tmp = np.empty_like(p)
    for t in range(Bt.shape[0]):                                     # in place: the same two rounded operations per term
        np.multiply(a[..., None, 32 * t:32 * t + 32], Bt[t], out=tmp)
        np.add(p, tmp, out=p)
    return _butterfly(p)


def canon_self_dot(X):
    """dot(x, x) of every row of X [n, d] -> [n]."""
    X = _pad32(X)
    p = np.zeros((X.shape[0], 32), dtype=np.float64)
    for t in range(X.shape[1] // 32):
        c = X[:, 32 * t:32 * t + 32]
        p = p + c * c
    return _butterfly(p)


def canon_normalize(X):
    X = np.asarray(X, dtype=np.float64)
    ss = canon_self_dot(X)
    nrm = np.sqrt(ss)
    return np.where(ss[:, None] > 0, X / np.where(nrm > 0, nrm, 1.0)[:, None], X)


def exact_topk(X, Y, k, thr=0.0, self_match=False, rows=None, normalized=False, block=8):
    """Canonical top-k of the rows `rows` (default: all) of X against Y.  Returns (idx int32 [r, k], val float64 [r, k])."""
    Xn = np.asarray(X, dtype=np.float64) if normalized else canon_normalize(X)
    Yn = np.asarray(Y, dtype=np.float64) if normalized else canon_normalize(Y)
    rows = np.arange(Xn.shape[0]) if rows is None else np.asarray(rows)
    idx = np.full((len(rows), k), -1, dtype=np.int32); val = np.zeros((len(rows), k), dtype=np.float64)
    Yt = _by_term(Yn)
    for b0 in range(0, len(rows), block):
        rb = rows[b0:b0 + block]
        S = canon_dot(Xn[rb], Yn, Yt)
        for r, (i, s) in enumerate(zip(rb, S)):
            ok = s > thr
            if self_match and i < len(s):
                ok[i] = False
            js = np.nonzero(ok)[0]
            order = js[np.lexsort((js, -s[js]))][:k]
            idx[b0 + r, :len(order)] = order; val[b0 + r, :len(order)] = s[order]
    return idx, val
