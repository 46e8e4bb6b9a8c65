"""CPU oracle and input generators for bit-exact tests of the Embeddings bf16 mode (K4, precision="bf16").

Grid rows.  Every entry is m / 8 with an integer |m| <= 8, and a row has at most 256 non-zeros.  Such entries are exact in
bf16, fp16 and fp64; every product is a multiple of 2^-6 of magnitude <= 1, so every partial sum of a dot product, in any
order, is a multiple of 2^-6 of magnitude <= 2^8: 14 significant bits.  An fp32 accumulator that keeps at least 16 bits per
addition therefore returns the exact rational score, whatever order and alignment it uses.  The oracle scores the pairs
as (M_x @ M_y^T) / 64 in fp64 on the integer grid, which is exact.

Top-k rule of the bf16 kernels (dense.py `sel_thr`, DESIGN.md 4.7): a pair (i, j) is eligible iff score > float32(thr) and,
in a self-match, from_base + i != to_base + j; rank by (score desc, global index asc); empty slots are (-1, 0.0).

Power-of-4 rows.  Rows of 8 non-zeros whose integer squares sum to 64, e.g. (7, 3, 1, 1, 1, 1, 1, 1): their l2
normalisation is the row / 8 exactly, in bf16, fp16 and fp64 alike, so both precisions of Embeddings score them exactly."""
import numpy as np

GRID = 8                          # entries m / GRID
NNZ_MAX = 256                     # non-zeros per row: the bit budget above

# integer rows of 8 entries whose squares sum to 64 (norm 8)
POW4_PATTERNS = [(7, 3, 1, 1, 1, 1, 1, 1), (5, 5, 3, 1, 1, 1, 1, 1), (6, 2, 2, 2, 2, 2, 2, 2), (4, 4, 4, 4, 0, 0, 0, 0),
                 (4, 4, 4, 2, 2, 2, 2, 0), (6, 4, 2, 2, 2, 0, 0, 0), (8, 0, 0, 0, 0, 0, 0, 0)]


def grid_rows(rng, n, d, nnz=None, zero_rows=()):
    """int8 [n, d] grid numerators (entries / 8 are the rows): per row a random number of non-zeros up to min(d, 256)
    (or exactly `nnz`), values uniform in -8..8 without 0.  Rows listed in `zero_rows` are all zero."""
    cap = min(d, NNZ_MAX)
    M = np.zeros((n, d), dtype=np.int8)
    for i in range(n):
        c = int(rng.integers(1, cap + 1)) if nnz is None else min(int(nnz), cap)
        cols = rng.choice(d, c, replace=False)
        v = rng.integers(1, GRID + 1, c) * rng.choice(np.array([-1, 1]), c)
        M[i, cols] = v
    M[list(zero_rows)] = 0
    return M


def tied_rows(rng, n, d, pool=6, frac=0.5, at=()):
    """Grid numerators [n, d] in which a small pool of distinct rows repeats at scattered positions (about `frac` of the rows,
    always at the positions `at`), so that every row scored against them sees runs of exactly tied scores."""
    M = grid_rows(rng, n, d)
    P = grid_rows(rng, pool, d)
    pos = np.nonzero(rng.random(n) < frac)[0]
    pos = np.union1d(pos, [p for p in at if 0 <= p < n]).astype(np.int64)
    M[pos] = P[rng.integers(0, pool, len(pos))]
    return M


def as_float(M, dtype=np.float32):
    return M.astype(dtype) / GRID


def grid_scores(Mx, My):
    """Exact fp64 scores of the grid rows Mx / 8 against My / 8."""
    return (Mx.astype(np.float64) @ My.astype(np.float64).T) / (GRID * GRID)


def topk(S, k, thr=0.0, self_match=False, from_base=0, to_base=0, f32_thr=True):
    """Top-k of the score matrix S [n, m] under the rule of the module docstring.  f32_thr: compare with float32(thr), as
    the bf16 kernels do; else with thr (the exact mode).  Returns (idx int32 [n, k] global to-indices, val float64 [n, k])."""
    S = np.asarray(S, dtype=np.float64)
    n, m = S.shape
    t = float(np.float32(thr)) if f32_thr else float(thr)
    ok = S > t
    if self_match:
        i = np.arange(n) + from_base - to_base                      # local to-column of each row's diagonal
        r = np.nonzero((i >= 0) & (i < m))[0]
        ok[r, i[r]] = False
    key = np.where(ok, -S, np.inf)                                  # ascending key; a stable sort keeps index order in ties
    order = np.argsort(key, axis=1, kind="stable")[:, :k]
    kk = order.shape[1]
    good = np.take_along_axis(ok, order, 1)
    idx = np.full((n, k), -1, dtype=np.int32)
    val = np.zeros((n, k), dtype=np.float64)
    idx[:, :kk] = np.where(good, order + to_base, -1)
    val[:, :kk] = np.where(good, np.take_along_axis(S, order, 1), 0.0)
    return idx, val


def split_ranges(n_to, n_splits, tile=128):
    """The to-column ranges of K4's splits: 128-wide tiles, ceil(tiles / n_splits) tiles per split (some may be empty)."""
    tiles = (n_to + tile - 1) // tile
    per = (tiles + n_splits - 1) // n_splits
    return [(min(n_to, s * per * tile), min(n_to, (s + 1) * per * tile)) for s in range(n_splits)]


def bounded_overflow(S, k, thr, cap, n_splits, self_match=False, from_base=0, to_base=0, list_k=16):
    """Rows the bf16 top_n > 32 path (dense.dense_topn_bounded, DESIGN.md 4.7) must re-run, for one chunk of from-rows and
    n_splits bound splits: tau_i = the k-th best of the union of the splits' top-`list_k` eligible entries (no bound with fewer
    than k), and the threshold pass keeps every column with score >= tau_i and score > float32(thr), the diagonal included.
    Returns the number of rows whose count exceeds cap."""
    S = np.asarray(S, dtype=np.float64)
    n, m = S.shape
    t = float(np.float32(thr))
    tau = np.full(n, -np.inf)
    for i in range(n):
        union = []
        for lo, hi in split_ranges(m, n_splits):
            if lo >= hi:
                continue
            ii, v = topk(S[i:i + 1, lo:hi], list_k, thr, self_match, from_base + i, to_base + lo)
            union.extend(v[0][ii[0] >= 0].tolist())
        if len(union) >= k:
            tau[i] = sorted(union, reverse=True)[k - 1]
    count = ((S >= tau[:, None]) & (S > t)).sum(1)
    return int((count > cap).sum())


# ---- bf16 rounding -------------------------------------------------------------------------------------------------------------

def bf16_bits_rne(x32):
    """uint16 bits of the round-to-nearest-even bf16 of float32 values (finite)."""
    b = np.ascontiguousarray(x32, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def bf16_to_f64(bits):
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def unit_rows(X):
    """x / ||x|| in fp64 at any scale (each row first scaled by the power of two of its largest |x|); zero rows stay zero."""
    X = np.asarray(X, dtype=np.float64)
    m = np.abs(X).max(1)
    _, e = np.frexp(np.where(m > 0, m, 1.0))
    Xs = np.ldexp(X, -e[:, None])                                   # exact, but for elements below 2^-1074 of the largest
    nrm = np.sqrt((Xs * Xs).sum(1))
    return np.where((m > 0)[:, None], Xs / np.where(nrm > 0, nrm, 1.0)[:, None], X)


def bf16_neighbours(t):
    """(lo, hi): the bf16 values with lo <= t <= hi adjacent (equal when t is one), for fp64 t in bf16's normal range."""
    t = np.asarray(t, dtype=np.float64)
    _, p = np.frexp(t)                                              # |t| = f 2^p, f in [0.5, 1): bf16 spacing 2^(p - 8)
    ulp = np.ldexp(1.0, p - 8)
    q = t / ulp                                                     # exact: a power-of-two scaling
    return np.floor(q) * ulp, np.ceil(q) * ulp


def pow4_rows(rng, n, d, scale_exp=None):
    """float64 [n, d]: each row a power-of-4 pattern with random signs, order and columns (d >= 8), times 2^e for a random
    e in -4..4 (or scale_exp).  Its l2 normalisation is pattern / 8 exactly."""
    X = np.zeros((n, d))
    for i in range(n):
        p = np.array(POW4_PATTERNS[rng.integers(len(POW4_PATTERNS))], dtype=np.float64)
        p = rng.permutation(p) * rng.choice(np.array([-1.0, 1.0]), 8)
        e = int(rng.integers(-4, 5)) if scale_exp is None else scale_exp
        X[i, rng.choice(d, 8, replace=False)] = np.ldexp(p, e)
    return X
