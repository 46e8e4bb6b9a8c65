"""The two CPU oracles agree on score cutoffs that land on achieved scores (no GPU needed).

oracle.native (C, the all-pairs arg-best the GPU tests of K3 compare with) and oracle.fuzz (rapidfuzz 3.x restated) must
apply rapidfuzz's two-step cutoff of fuzz.ratio the same way: ns = 1 - indel/(|a|+|b|) is kept only if ns >= c/100, and
extractOne then keeps the score ns*100 only if it is >= c.  The two steps disagree whenever (ns*100)/100 != ns; the pairs
where they do ("boundary pairs") are generated here for the other scorers too and pinned as known answers, so the GPU tests
that use the same generator are known to contain them."""
import functools
import math

import numpy as np
import pytest

import cutoff_cases as cc
import lcs_oracle
from oracle import fuzz as ofuzz
from oracle import native


@pytest.fixture(scope="module", autouse=True)
def c_lcs():
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ofuzz, "lcs_len", functools.lru_cache(maxsize=None)(lcs_oracle.lcs_len))
        yield


# ---- fuzz.ratio: every (|a|, |b|, lcs) with lengths 1..60 at every cutoff of the grid and at its own score ---------------------
def test_ratio_oracles_agree_at_every_cutoff():
    """Both oracles compute ratio from d = |a|+|b|-2*lcs and m = |a|+|b| alone, so every triple is represented by one pair per
    (m, d): |b| = m//2, |a| = m - |b|.  Per |b| one C call scores all its pairs against b = "a"*|b| at one cutoff."""
    reps = {}
    for la, lb, l in cc.ratio_triples(60):
        m = la + lb
        reps.setdefault((m, m - 2 * l), None)
    groups = {}
    for m, d in reps:
        lb = m // 2
        la, l = m - lb, (m - d) // 2
        groups.setdefault(lb, []).append(("a" * l + "b" * (la - l), cc.ratio_ns(la, lb, l)))
    grid = cc.cutoff_grid()
    n_boundary = n_checked = 0
    for lb, rows in groups.items():
        b = "a" * lb
        frm = [a for a, _ in rows]
        own = sorted({c for _, ns in rows for c in cc.neighbours(ns * 100.0)})
        n_boundary += sum(cc.is_boundary_score(ns) for _, ns in rows)
        for c in grid + own:
            bi, bs, _ = native.editdist_argbest(frm, [b], "ratio", score_cutoff=c)
            for r, a in enumerate(frm):
                e = ofuzz.extract_one(a, [b], ofuzz.ratio, c)
                got = None if bi[r] < 0 else (b, float(bs[r]), int(bi[r]))
                assert got == e, (len(a), lb, ofuzz.lcs_len(a, b), c, got, e)
                n_checked += 1
    assert n_boundary > 100 and n_checked > 1_000_000


def test_ratio_known_boundary_pair():
    """LCS 17 of 25 + 25 code points: ns = 0.6799999999999999, ns*100 = 68.0, and 68.0/100 = 0.68 > ns."""
    a, b = cc.ratio_strings(25, 25, 17)
    assert ofuzz.ratio(a, b) == 68.0 and cc.is_boundary_score(cc.ratio_ns(25, 25, 17))
    below = math.nextafter(68.0, 0)
    assert ofuzz.extract_one(a, [b], ofuzz.ratio, 68.0) is None
    assert ofuzz.extract_one(a, [b], ofuzz.ratio, below) == (b, 68.0, 0)
    bi, bs, _ = native.editdist_argbest([a], [b], "ratio", score_cutoff=68.0)
    assert bi.tolist() == [-1] and bs.tolist() == [0.0]
    bi, bs, _ = native.editdist_argbest([a], [b], "ratio", score_cutoff=below)
    assert bi.tolist() == [0] and bs.tolist() == [68.0]
    # the matchers' 0..1 cutoff 0.68 reaches the scorer as 68.0
    assert 0.68 * 100 == 68.0


def test_norm_lev_cutoff_is_one_test():
    """Levenshtein.normalized_similarity has no /100 step: a cutoff equal to the score keeps the pair."""
    for a, b in (("abcdefg", "abcxefy"), ("kitten", "sitting"), ("a" * 17 + "b" * 8, "a" * 25)):
        bi, s, _ = native.editdist_argbest([a], [b], "norm_lev")
        bi2, s2, _ = native.editdist_argbest([a], [b], "norm_lev", score_cutoff=float(s[0]))
        assert bi2.tolist() == [0] and s2.tolist() == s.tolist()
        bi3, _, _ = native.editdist_argbest([a], [b], "norm_lev", score_cutoff=math.nextafter(float(s[0]), 2.0))
        assert bi3.tolist() == [-1]


# ---- the other scorers: seeded boundary pairs --------------------------------------------------------------------------------
BOUNDARY_SCORERS = ["partial_ratio", "token_sort_ratio", "WRatio", "QRatio", "token_ratio", "partial_token_sort_ratio",
                    "partial_token_set_ratio", "partial_token_ratio"]


@pytest.mark.parametrize("scorer", BOUNDARY_SCORERS)
def test_generator_finds_boundary_pairs(scorer):
    pairs = cc.boundary_pairs(scorer, 8, seed=1)
    assert len(pairs) == 8
    fn = ofuzz.SCORERS[scorer]
    for a, b, s in pairs:
        assert fn(a, b, 0) == s and fn(a, b, s) == 0
        assert fn(a, b, math.nextafter(s, 0)) == s                 # one ulp lower keeps it
        assert ofuzz.extract_one(a, [b], fn, s) is None
        assert ofuzz.extract_one(a, [b], fn, math.nextafter(s, 0)) == (b, s, 0)


def test_token_set_ratio_has_no_boundary_pairs():
    """token_set_ratio's parts test score >= cutoff once (100 - 100*dist/lensum, no /100 step): the generator finds none, and a
    cutoff equal to the score keeps every pair."""
    assert cc.boundary_pairs("token_set_ratio", 1, seed=1, max_tries=3000) == []
    rng = np.random.default_rng(2)
    for _ in range(500):
        a = "".join(rng.choice(list("ab "), rng.integers(1, 30))); b = "".join(rng.choice(list("ab "), rng.integers(1, 30)))
        s = ofuzz.token_set_ratio(a, b)
        assert ofuzz.token_set_ratio(a, b, s) == s


# known answers: a cutoff equal to the score rejects the pair, one ulp below keeps it
KNOWN = [
    ("partial_ratio", "cbbcaaacb", "bbaacaccbaaabbbaaaacaacabccccbbc", 77.77777777777779),
    ("partial_ratio", "acbbbcbacaacbaabcbc", "aaccaacbb", 77.77777777777779),
    ("token_sort_ratio", "a bb a bb a  baba a", " bbb a b  aaaa ba aa  ", 77.77777777777779),
    ("token_sort_ratio", "aaa   aa", " bab aa aa  aba b abbaa b ", 41.379310344827594),
    ("WRatio", "cb aca", "cca  a bab  cbaccbc cabbb a", 75.00000000000001),
    ("WRatio", "cbacccaabb babba cb b  bcaaaa", " babb ccaa", 66.50000000000001),
    ("QRatio", "bbcbbcccabaaabaabbcbaaaba", "ababbcbaaabacbacacbbbcaba", 68.0),
    ("partial_token_ratio", " bcbaaabb bbacac a ", "ba bbcbacab", 77.77777777777779),
]


@pytest.mark.parametrize("scorer,a,b,s", KNOWN)
def test_known_boundary_pairs(scorer, a, b, s):
    fn = ofuzz.SCORERS[scorer]
    assert fn(a, b) == s
    assert fn(a, b, s) == 0
    assert fn(a, b, math.nextafter(s, 0)) == s


# ---- the matchers' 0..1 cutoffs ------------------------------------------------------------------------------------------------
def test_matcher_rescales_unit_metric_cutoffs(monkeypatch):
    """RapidFuzz takes score_cutoff u in 0..1 and hands u*100 to the 0..100 scorers; for the 0..1 metrics (levenshtein, osa, dl)
    it hands on (u*100)/100, which is not always u.  This pins the current rescaling (it is not rapidfuzz's: the reference
    passes u*100 to every scorer)."""
    import torch
    from polyfuzz_b200 import editdist
    from polyfuzz_b200.matchers import _rapidfuzz
    seen = []

    def fake_argbest(from_list, to_list, metric, cutoff, **kw):
        seen.append((metric, cutoff))
        n = len(from_list)
        return torch.full((n,), -1, dtype=torch.int32), torch.zeros(n, dtype=torch.float64), torch.full((n,), -1, dtype=torch.int32)

    monkeypatch.setattr(editdist, "edit_argbest", fake_argbest)
    u = next(k / 1000 for k in range(1, 1000) if (k / 1000 * 100) / 100 != k / 1000)
    for scorer, metric in (("levenshtein", "norm_lev"), ("osa", "norm_osa"), ("dl", "norm_dl"), ("ratio", "ratio")):
        seen.clear()
        m = _rapidfuzz.RapidFuzz(scorer=scorer, score_cutoff=u).match(["x"], ["y"])
        assert m.To.tolist() == [None] and m.Similarity.tolist() == [0.0]
        exp = (u * 100) / 100 if metric != "ratio" else u * 100
        assert seen == [(metric, exp)]
    assert (u * 100) / 100 != u
