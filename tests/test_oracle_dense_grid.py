"""CPU tests (no GPU) of tests/dense_grid_oracle.py: the grid generators keep the bit budget and score exactly, the power-of-4
rows normalise exactly in bf16 and fp16, the top-k oracle follows the bf16 kernels' rule on hand-made cases, and the bf16
helpers round as bf16 does."""
import os
import sys
from fractions import Fraction

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dense_grid_oracle as G                                       # noqa: E402


def test_grid_rows_respect_the_bit_budget():
    rng = np.random.default_rng(0)
    for d in (8, 200, 1024, 4096):
        M = G.grid_rows(rng, 64, d, zero_rows=[3])
        assert M.dtype == np.int8 and np.abs(M).max() <= 8
        nnz = (M != 0).sum(1)
        assert nnz.max() <= min(d, 256) and nnz[3] == 0 and (np.delete(nnz, 3) >= 1).all()
        # |sum of products| <= 256 * 64 (numerators), so every partial sum is a multiple of 2^-6 below 2^8: 14 bits
        A = np.abs(M.astype(np.int64))
        assert (A @ A.T).max() <= 256 * 64
        T = G.tied_rows(rng, 500, d, at=(127, 128, 499))
        assert np.abs(T).max() <= 8 and ((T != 0).sum(1) <= 256).all()
        assert len({T[j].tobytes() for j in (127, 128, 499)}) <= 6
        assert len({r.tobytes() for r in T}) < 500                     # the pool repeats


def test_grid_rows_are_exact_in_bf16_and_fp16():
    rng = np.random.default_rng(1)
    X = G.as_float(G.grid_rows(rng, 50, 72))
    for dt in (torch.bfloat16, torch.float16):
        assert np.array_equal(torch.from_numpy(X).to(dt).float().numpy(), X)


def test_grid_scores_equal_exact_integer_arithmetic():
    rng = np.random.default_rng(2)
    Mx = G.grid_rows(rng, 40, 300)
    My = G.tied_rows(rng, 60, 300)
    S = G.grid_scores(Mx, My)
    I = Mx.astype(np.int64) @ My.astype(np.int64).T
    assert np.array_equal(S * 64, I.astype(np.float64)) and np.array_equal(S, I / 64.0)
    for i, j in ((0, 0), (3, 17), (39, 59)):
        exact = sum(Fraction(int(a), 8) * Fraction(int(b), 8) for a, b in zip(Mx[i], My[j]))
        assert Fraction(S[i, j]) == exact
    # in float32 too: the scores (and the partial sums) are exact in fp32
    assert np.array_equal(S.astype(np.float32).astype(np.float64), S)


def test_pow4_rows_normalise_exactly():
    rng = np.random.default_rng(3)
    for p in G.POW4_PATTERNS:
        assert sum(v * v for v in p) == 64
    X = G.pow4_rows(rng, 200, 64)
    U = G.unit_rows(X)
    assert np.array_equal(U * 8, np.round(U * 8)) and ((U != 0).sum(1) <= 8).all()
    assert np.array_equal(np.linalg.norm(U, axis=1), np.ones(200))
    for dt in (torch.bfloat16, torch.float16, torch.float64):
        assert np.array_equal(torch.from_numpy(U).to(dt).double().numpy(), U)
    # scores of the normalised rows are multiples of 1/64: exact in fp32
    S = U @ U.T
    assert np.array_equal(S * 64, np.round(S * 64)) and np.array_equal(S.astype(np.float32).astype(np.float64), S)


def test_topk_ties_by_index_and_fill():
    S = np.array([[0.5, 1.0, 0.5, 1.0, 0.25, 0.5]])
    i, v = G.topk(S, 4, 0.0)
    assert i.tolist() == [[1, 3, 0, 2]] and v.tolist() == [[1.0, 1.0, 0.5, 0.5]]
    i, v = G.topk(S, 8, 0.3)
    assert i.tolist() == [[1, 3, 0, 2, 5, -1, -1, -1]] and v.tolist() == [[1.0, 1.0, 0.5, 0.5, 0.5, 0.0, 0.0, 0.0]]
    i, v = G.topk(S, 3, 0.0, to_base=100)
    assert i.tolist() == [[101, 103, 100]]
    i, v = G.topk(np.zeros((2, 3)), 2, 0.0)
    assert i.tolist() == [[-1, -1], [-1, -1]] and v.tolist() == [[0.0, 0.0], [0.0, 0.0]]
    i, v = G.topk(np.array([[0.0, -0.5, 0.0]]), 3, -1.0)                 # negative threshold: zeros and negatives eligible
    assert i.tolist() == [[0, 2, 1]] and v.tolist() == [[0.0, 0.0, -0.5]]


def test_topk_strict_threshold_in_float32():
    S = np.array([[0.5, 0.75, 0.5 + 2.0 ** -6]])
    assert G.topk(S, 3, 0.5)[0].tolist() == [[1, 2, -1]]                    # a score equal to the threshold is dropped
    s = 0.5 + 2.0 ** -6
    thr = s - 2.0 ** -30                                                    # float32(thr) == s: s is dropped as well
    assert float(np.float32(thr)) == s
    assert G.topk(S, 3, thr)[0].tolist() == [[1, -1, -1]]
    assert G.topk(S, 3, thr, f32_thr=False)[0].tolist() == [[1, 2, -1]]     # the exact mode compares in fp64


def test_topk_diagonal_with_bases():
    S = np.full((3, 4), 0.5)
    assert G.topk(S, 4, 0.0, self_match=True)[0].tolist() == [[1, 2, 3, -1], [0, 2, 3, -1], [0, 1, 3, -1]]
    # from-block starting at global row 2 against the whole to-list: the diagonal is column 2 + i
    assert G.topk(S, 4, 0.0, self_match=True, from_base=2)[0].tolist() == [[0, 1, 3, -1], [0, 1, 2, -1], [0, 1, 2, 3]]
    # to-shard starting at global column 2: row i's diagonal is local column i - 2
    assert G.topk(S, 4, 0.0, self_match=True, to_base=2)[0].tolist() == [[2, 3, 4, 5], [2, 3, 4, 5], [3, 4, 5, -1]]


def test_split_ranges_and_overflow_count():
    assert G.split_ranges(300, 2) == [(0, 256), (256, 300)]
    assert G.split_ranges(300, 3) == [(0, 128), (128, 256), (256, 300)]
    assert G.split_ranges(129, 4) == [(0, 128), (128, 129), (129, 129), (129, 129)]
    S = np.zeros((2, 300))
    S[0, :50] = 1.0                                                         # 16 listed (split 0) < 33: no bound, count 50
    S[1, :5] = 1.0                                                          # fewer than k eligible: no bound, count 5
    assert G.bounded_overflow(S, 33, 0.0, 40, 2) == 1
    assert G.bounded_overflow(S, 33, 0.0, 50, 2) == 0
    assert G.bounded_overflow(S, 33, -1.0, 100, 2) == 2                     # threshold -1: 16 + 16 listed < 33, no bound: 300 each


def test_bf16_helpers():
    x = np.array([1.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -2.5, 2.0 ** -130, 0.0, -0.0, 3.0e38], dtype=np.float32)
    want = torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(G.bf16_bits_rne(x), want)
    assert np.array_equal(G.bf16_to_f64(want), torch.from_numpy(x).to(torch.bfloat16).double().numpy())
    t = np.array([1.0, 1.0 + 2.0 ** -9, -(1.0 + 2.0 ** -9), 0.75 + 2.0 ** -12, 2.0 ** -100 * 1.001, 0.0])
    lo, hi = G.bf16_neighbours(t)
    assert lo.tolist() == [1.0, 1.0, -(1.0 + 2.0 ** -7), 0.75, 2.0 ** -100, 0.0]
    assert hi.tolist() == [1.0, 1.0 + 2.0 ** -7, -1.0, 0.75 + 2.0 ** -8, 2.0 ** -100 * (1 + 2.0 ** -7), 0.0]
    rng = np.random.default_rng(4)
    t = rng.standard_normal(10_000) * np.ldexp(1.0, rng.integers(-100, 100, 10_000))
    lo, hi = G.bf16_neighbours(t)
    b = torch.from_numpy(t).to(torch.bfloat16).double().numpy()           # nearest: one of the two
    assert ((b == lo) | (b == hi)).all() and (lo <= t).all() and (t <= hi).all() and ((hi - lo) <= np.abs(t) * 2.0 ** -7).all()


def test_unit_rows_at_any_scale():
    rng = np.random.default_rng(5)
    X = rng.standard_normal((20, 30))
    U = G.unit_rows(X)
    np.testing.assert_allclose(U, X / np.linalg.norm(X, axis=1, keepdims=True), rtol=1e-15, atol=0)
    for e in (-900, 900, 1000):
        assert np.array_equal(G.unit_rows(np.ldexp(X, e)), U)
    Z = np.zeros((2, 5)); Z[1, 3] = -7.0
    assert G.unit_rows(Z).tolist() == [[0.0] * 5, [0.0, 0.0, 0.0, -1.0, 0.0]]
