"""Bit-exact GPU tests of the Embeddings bf16 mode (K4): the top-k kernels on inputs whose fp32 scores cannot depend on the
order of accumulation, and the row staging (`dense.to_bf16_rows`) against a plain numpy reference.

Assumption behind the top-k tests: the H100's bf16 wgmma with fp32 accumulation is exact when every partial sum fits in
about 16 significant bits.  The grid rows of tests/dense_grid_oracle.py (entries m / 8, |m| <= 8, at most 256 non-zeros per
row) keep every partial sum of every dot product a multiple of 2^-6 of magnitude <= 2^8, i.e. within 14 bits, so the kernel's
fp32 score must equal the exact score, whatever its summation order or alignment.  The bf16 tensors go straight to
`dense.dense_topk` / `dense.dense_topn_bounded` (no staging), and idx / val must equal the numpy oracle with ==: eligible
iff score > float32(min_similarity) and not the diagonal of a self-match, ranked by (score desc, index asc), empty slots
(-1, 0.0).  On a mismatch the message gives the kernel's and the exact score of the pair, so that a failure can be told
apart from an accumulation that kept fewer bits than assumed.

The to-sides repeat a small pool of rows at scattered positions (columns 127 / 128, both columns of an 8j + {0, 1} pair,
split boundaries, the last row), so each from-row has runs of exactly tied scores longer than k that straddle tiles,
splits and the lanes of a quad, and the k-th rank falls inside a tie."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dense_grid_oracle as G                                       # noqa: E402

pytestmark = pytest.mark.gpu

K_TOPK = (1, 4, 5, 10, 11, 16, 17, 32)                              # every KMAX instantiation (4 / 10 / 16 / 32) and its edges
K_BOUNDED = (33, 64, 300)


def _dev(M):
    """grid numerators -> device bf16 rows (exact)"""
    return torch.from_numpy(G.as_float(M)).to("cuda").to(torch.bfloat16)


def _default_splits(n_from, n_to):
    from polyfuzz_b200 import dense
    mb, nt = (n_from + 127) // 128, (n_to + 127) // 128
    return max(1, min(nt, (2 * dense.SM_COUNT + mb - 1) // mb))


def _tie_positions(n_to, n_from):
    """to-columns that must hold pool rows: tile and quad-pair edges, the last row, the boundaries of the default splits"""
    at = {0, 1, 126, 127, 128, 129, 8 * 17, 8 * 17 + 1, 8 * 37 + 6, 8 * 37 + 7, n_to - 2, n_to - 1}
    for s in (_default_splits(n_from, n_to), 3):
        for lo, _ in G.split_ranges(n_to, s)[1:]:
            at.update((lo - 1, lo))
    return sorted(p for p in at if 0 <= p < n_to)


def _eq(got, exp, S, ctx, to_base=0):
    """kernel (idx, val) == oracle (idx, val); on a mismatch report the first differing slot with the exact scores"""
    gi, gv = got[0].cpu().numpy(), got[1].cpu().numpy()
    oi, ov = exp
    assert gi.shape == oi.shape, (ctx, gi.shape, oi.shape)
    bad = np.nonzero((gi != oi).any(1) | (gv != ov).any(1))[0]
    if len(bad):
        r = int(bad[0])
        c = int(np.nonzero((gi[r] != oi[r]) | (gv[r] != ov[r]))[0][0])
        j = int(gi[r, c]) - to_base
        exact = float(S[r, j]) if 0 <= j < S.shape[1] else None
        raise AssertionError(f"{ctx}: {len(bad)} rows differ; row {r} slot {c}: kernel (idx {gi[r, c]}, score {gv[r, c]!r}, exact score "
                             f"of that pair {exact!r}), oracle (idx {oi[r, c]}, score {ov[r, c]!r}); "
                             f"kernel row {gi[r, :c + 3].tolist()} / {gv[r, :c + 3].tolist()}, oracle row {oi[r, :c + 3].tolist()}")


def _cut(o, k):
    return o[0][:, :k], o[1][:, :k]


def _attained(S, lo=2.0 ** -5):
    """an attained score s >= 2^-5 that is not a power of two: thr = s - 2^-30 rounds to s in fp32"""
    v = np.unique(S[S >= lo])
    v = v[np.frexp(v)[0] != 0.5]
    return float(v[len(v) // 2])


SHAPES = [(1, 1, 8), (127, 3, 16), (128, 127, 56), (129, 128, 64), (383, 129, 72), (1000, 3000, 200), (383, 2500, 1024),
          (129, 1200, 4096), (1, 5000, 8)]


@pytest.mark.parametrize("two_cta", ["0", "1"])
@pytest.mark.parametrize("n_from,n_to,d", SHAPES)
def test_topk_grid_equals_oracle(n_from, n_to, d, two_cta, monkeypatch):
    """Every k instantiation, n_splits None / 1 / the maximum, thresholds 0 and -1 (negative scores), then a threshold on
    an attained score and just below it (strict >, compared in fp32), through dense_topk (k <= 32) and the bounded path."""
    from polyfuzz_b200 import dense
    monkeypatch.setenv("PFZ_K4_2CTA", two_cta)
    rng = np.random.default_rng(n_from * 1009 + n_to * 7 + d)
    My = G.tied_rows(rng, n_to, d, at=_tie_positions(n_to, n_from))
    Mx = G.grid_rows(rng, n_from, d, zero_rows=[n_from // 2] if n_from > 2 else [])
    if n_from > 8:
        Mx[3] = My[n_to - 1]; Mx[5, :] = 0; Mx[5, :4] = 1              # a row equal to a to-row; a row with few eligible to-rows
    S = G.grid_scores(Mx, My)
    x, y = _dev(Mx), _dev(My)
    n_tiles = (n_to + 127) // 128
    for thr in (0.0, -1.0):
        o = G.topk(S, max(K_BOUNDED), thr)
        if n_to >= 1000 and n_from >= 100:                           # the inputs do what they are for: the cut falls in a tie
            assert all(((o[1][:, k - 1] == o[1][:, k]) & (o[0][:, k] >= 0)).any() for k in K_TOPK + K_BOUNDED[:2])
        for splits in (None, 1, n_tiles):
            for k in K_TOPK:
                _eq(dense.dense_topk(x, y, k, thr, n_splits=splits), _cut(o, k), S, (thr, splits, k))
        for k in K_BOUNDED:
            _eq(dense.dense_topk(x, y, k, thr), _cut(o, k), S, (thr, "bounded", k))
            _eq(dense.dense_topn_bounded(x, y, k, thr, n_splits=n_tiles)[:2], _cut(o, k), S, (thr, "bounded", n_tiles, k))
    if (S >= 2.0 ** -5).any():
        s = _attained(S)
        for thr in (s, s - 2.0 ** -30):
            assert float(np.float32(thr)) == s
            o = G.topk(S, 64, thr)
            assert not (o[1][o[0] >= 0] <= s).any()
            for k in (5, 32, 33, 64):
                _eq(dense.dense_topk(x, y, k, thr), _cut(o, k), S, (thr, k))


@pytest.mark.parametrize("two_cta", ["0", "1"])
def test_bounded_overflow_count_and_rerun(two_cta, monkeypatch):
    """A small candidate capacity: rows overflow and take the re-run, the result still equals the oracle, and the number of
    re-run rows is the number whose threshold-pass candidates (score >= the row's bound, score > float32(thr)) exceed cap.
    In the sparse cases most rows have fewer than k eligible to-rows (no bound) and thousands scoring exactly the threshold,
    which the threshold pass must not keep."""
    from polyfuzz_b200 import dense
    monkeypatch.setenv("PFZ_K4_2CTA", two_cta)
    rng = np.random.default_rng(11)
    cases = [(G.grid_rows(rng, 300, 64), G.tied_rows(rng, 3000, 64, pool=3, frac=0.3, at=_tie_positions(3000, 300)), 33, 40, 0.0),
             (G.grid_rows(rng, 300, 200, nnz=2), G.grid_rows(rng, 3000, 200, nnz=2), 33, 40, 0.0),
             (G.grid_rows(rng, 200, 200, nnz=3), G.grid_rows(rng, 3000, 200, nnz=3), 64, 100, 0.0)]
    n_over_total = 0
    for Mx, My, k, cap, thr in cases:
        S = G.grid_scores(Mx, My)
        x, y = _dev(Mx), _dev(My)
        n_tiles = (My.shape[0] + 127) // 128
        for n_splits in (4, n_tiles):
            s = max(1, min(n_tiles, max(-(-2 * k // 16), n_splits)))   # the bound pass's split count (dense_topn_bounded)
            idx, val, n_over = dense.dense_topn_bounded(x, y, k, thr, n_splits=n_splits, cap=cap)
            _eq((idx, val), G.topk(S, k, thr), S, (k, cap, n_splits))
            assert n_over == G.bounded_overflow(S, k, thr, cap, s), (k, cap, n_splits, n_over)
            n_over_total += n_over
    assert n_over_total > 0


@pytest.mark.parametrize("two_cta", ["0", "1"])
def test_self_match_shards_and_blocks(two_cta, monkeypatch):
    """Self-match against to-shards (to_index_base) and from-blocks (from_index_base): each equals the oracle, and the
    merged shard lists equal the single call with ==.  Repeated rows tie with the (excluded) diagonal's score."""
    from polyfuzz_b200 import dense
    from polyfuzz_b200.distributed import merge_topk_any, shard_bounds
    monkeypatch.setenv("PFZ_K4_2CTA", two_cta)
    rng = np.random.default_rng(12)
    n = 2100
    M = G.tied_rows(rng, n, 64, pool=5, frac=0.3, at=_tie_positions(n, n))
    M[17] = 0
    S = G.grid_scores(M, M)
    y = _dev(M)
    bounds = [shard_bounds(n, 3, r) for r in range(3)]
    for thr in (0.0, -1.0):
        o = G.topk(S, 100, thr, self_match=True)
        for k in (1, 10, 32, 40, 100):
            single = dense.dense_topk(y, y, k, thr, self_match=True)
            _eq(single, _cut(o, k), S, ("self", thr, k))
            parts_i, parts_v = [], []
            for lo, hi in bounds:
                part = dense.dense_topk(y, y[lo:hi], k, thr, self_match=True, to_index_base=lo)
                _eq(part, G.topk(S[:, lo:hi], k, thr, self_match=True, to_base=lo), S[:, lo:hi], ("to-shard", lo, thr, k), to_base=lo)
                parts_i.append(part[0]); parts_v.append(part[1])
                blk = dense.dense_topk(y[lo:hi], y, k, thr, self_match=True, from_index_base=lo)
                _eq(blk, (o[0][lo:hi, :k], o[1][lo:hi, :k]), S[lo:hi], ("from-block", lo, thr, k))
            mi, mv = merge_topk_any(torch.stack(parts_i), torch.stack(parts_v), k)
            assert torch.equal(mi, single[0]) and torch.equal(mv, single[1]), (thr, k)


def _frame_lists(df):
    return {c: [None if (isinstance(v, float) and np.isnan(v)) else v for v in df[c].tolist()] for c in df.columns}


def test_matcher_pow4_rows_both_precisions_equal_the_oracle():
    """Rows whose normalisation is exact in bf16, fp16 and fp64: Embeddings(precision="bf16") and precision="fp64" return
    the same frames, equal to the oracle's top-n put through the reference's frame assembly."""
    from polyfuzz_b200 import Embeddings
    from oracle.assemble import assemble
    rng = np.random.default_rng(13)
    ef, et = G.pow4_rows(rng, 300, 64), G.pow4_rows(rng, 500, 64)
    ef[7] = 0.0
    frm = [f"from {i}" for i in range(len(ef))]
    to = [f"to {i}" for i in range(len(et))]
    unit = lambda X: X / np.where((X != 0).any(1), np.linalg.norm(X, axis=1), 1.0)[:, None]   # noqa: E731  (exact here)
    S2, S1 = unit(ef) @ unit(et).T, unit(ef) @ unit(ef).T
    for top_n in (1, 10, 40):
        for thr in (0.0, 0.5):
            for to_list, emb_to, S, sm in ((to, et, S2, False), (None, None, S1, True)):
                exp = _frame_lists(assemble(frm, to_list, *G.topk(S, top_n, thr, self_match=sm)))
                for precision in ("bf16", "fp64"):
                    df = Embeddings(min_similarity=thr, top_n=top_n, precision=precision).match(frm, to_list, ef, emb_to)
                    assert _frame_lists(df) == exp, (precision, top_n, thr, sm)


# ---- staging: dense.to_bf16_rows against numpy --------------------------------------------------------------------------------

def _staged(X, normalize):
    from polyfuzz_b200 import dense
    out, _ = dense.to_bf16_rows(X, normalize)
    return out.view(torch.int16).cpu().numpy().view(np.uint16)


def _inputs(rng, n, d, dtype):
    """Gaussian rows at per-row scales across the type's range, one-hot rows, zero rows, and exponents up to the limits"""
    X = rng.standard_normal((n, d))
    lim = 120 if dtype == np.float32 else 1000
    X *= np.ldexp(1.0, rng.integers(-lim, lim + 1, n))[:, None]
    X[0] = 0.0
    X[1] = 0.0; X[1, d // 2] = -3.0
    X[2] = 0.0; X[2, 0] = 2.0 ** (-140 if dtype == np.float32 else -1060)
    if d > 1:
        X[3, 0] = X[3, 1] * 2.0 ** -200                                 # an element far below the row's largest
    return X.astype(dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("d", [1, 7, 8, 13, 300, 768, 4096])
def test_staging_unnormalized_is_rne_of_fp32(d, dtype):
    rng = np.random.default_rng(d)
    n = 17_100 if d <= 13 else 300
    X = rng.standard_normal((n, d)) * np.ldexp(1.0, rng.integers(-140, 100, n))[:, None]
    X[0] = 0.0
    X = X.astype(dtype)
    got = _staged(X, False)
    d_pad = max(8, (d + 7) // 8 * 8)
    assert got.shape == (n, d_pad)
    with np.errstate(over="ignore"):
        assert np.array_equal(got[:, :d], G.bf16_bits_rne(X.astype(np.float32)))
    assert (got[:, d:] == 0).all() and (got[0] == 0).all()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("d", [1, 7, 8, 13, 300, 768, 4096])
def test_staging_normalized_is_faithful(d, dtype):
    """Every staged element is one of the two bf16 neighbours of x / ||x|| (fp64) wherever that is >= 2^-100 in magnitude;
    exact zeros stay +0, one-hot rows stage as exactly +-1, padding is +0.  > 17 000 rows wrap the grid-stride loop."""
    rng = np.random.default_rng(100 + d)
    n = 17_100 if d <= 13 else 400
    X = _inputs(rng, n, d, dtype)
    got = G.bf16_to_f64(_staged(X, True))
    d_pad = got.shape[1]
    assert d_pad == max(8, (d + 7) // 8 * 8)
    T = G.unit_rows(X)
    lo, hi = G.bf16_neighbours(T)
    big = np.abs(T) >= 2.0 ** -100
    g = got[:, :d]
    bad = big & (g != lo) & (g != hi)
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:3].tolist(), g[bad][:3], T[bad][:3])
    assert (g[T == 0] == 0).all() and (np.signbit(g[T == 0]) == np.signbit(T[T == 0])).all()
    assert (np.abs(g[~big]) <= 2.0 ** -99).all()
    assert (got[:, d:] == 0).all() and not np.signbit(got[:, d:]).any()
    assert got[1, d // 2] == -1.0 and got[2, 0] == 1.0 and (got[0] == 0).all()


def _grid128(rng, n, d):
    return rng.integers(-128, 129, (n, d)) / 128.0                    # power-of-two scalings of these are exact


@pytest.mark.parametrize("dtype,exps", [(np.float32, (-140, -100, -64, 64, 100, 126)), (np.float64, (-1000, -600, -300, 300, 600, 1000))])
def test_staging_invariant_under_powers_of_two(dtype, exps):
    """x and 2^e x stage to the same bits, and Embeddings() returns the same frames for them.  Lists every (what, d, e)
    that differs."""
    from polyfuzz_b200 import Embeddings
    rng = np.random.default_rng(21)
    bad = []
    for d in (13, 768):
        X = _grid128(rng, 700, d)
        X[5] = 0.0
        base = _staged(X.astype(dtype), True)
        bad += [("rows", d, e) for e in exps if not np.array_equal(_staged(np.ldexp(X, e).astype(dtype), True), base)]
    ef, et = _grid128(rng, 200, 64), _grid128(rng, 300, 64)
    frm = [f"f{i}" for i in range(len(ef))]
    to = [f"t{i}" for i in range(len(et))]
    m = Embeddings(min_similarity=0.0, top_n=5)
    ref = _frame_lists(m.match(frm, to, ef.astype(dtype), et.astype(dtype)))
    for e in exps:
        if _frame_lists(m.match(frm, to, np.ldexp(ef, e).astype(dtype), np.ldexp(et, e).astype(dtype))) != ref:
            bad.append(("frames", 64, e))
    assert not bad, str(bad)
