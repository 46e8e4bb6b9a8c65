"""CPU tests of the optimal string alignment (OSA, restricted Damerau-Levenshtein) metrics: the oracle's DP
(tests/osa_oracle.c) against a literal Python transcription of the definition and known values,
the scorer names and callables the matchers resolve to OSA, and the matchers' host logic with the kernels stubbed."""
import numpy as np
import pytest
import torch

import osa_oracle
from oracle import native


def osa_py(a, b):
    """The definition: Wagner-Fischer plus d[i][j] = min(d[i][j], d[i-2][j-2] + 1) for a swap of two adjacent characters."""
    la, lb = len(a), len(b)
    d = [[0] * (lb + 1) for _ in range(la + 1)]
    for i in range(la + 1):
        d[i][0] = i
    for j in range(lb + 1):
        d[0][j] = j
    for i in range(1, la + 1):
        for j in range(1, lb + 1):
            d[i][j] = min(d[i - 1][j] + 1, d[i][j - 1] + 1, d[i - 1][j - 1] + (a[i - 1] != b[j - 1]))
            if i > 1 and j > 1 and a[i - 1] == b[j - 2] and a[i - 2] == b[j - 1]:
                d[i][j] = min(d[i][j], d[i - 2][j - 2] + 1)
    return d[la][lb]


osa = osa_oracle.osa


def test_known_values():
    assert osa("ab", "ba") == 1
    assert osa("CA", "AC") == 1 and int(native.editdist_matrix(["CA"], ["AC"], "lev")[0, 0]) == 2
    assert osa("abc", "acb") == 1
    assert osa("abcdef", "badcfe") == 3 and int(native.editdist_matrix(["abcdef"], ["badcfe"], "lev")[0, 0]) == 4
    assert osa("kitten", "sitting") == 3
    assert osa("", "abc") == 3 and osa("abc", "") == 3 and osa("", "") == 0
    # restricted, not unrestricted Damerau-Levenshtein (which gives 2: CA -> AC -> ABC)
    assert osa("CA", "ABC") == 3
    _, bs, bd = osa_oracle.osa_argbest(["CA"], ["AC"], "norm_osa")
    assert bs[0] == 0.5 and bd[0] == 1
    _, bs, _ = osa_oracle.osa_argbest([""], [""], "norm_osa")
    assert bs[0] == 1.0


def test_oracle_equals_definition_on_random_pairs():
    rng = np.random.default_rng(11)
    frm, to = [], []
    for alpha, hi in (("ab", 10), ("abc", 14), ("abcdefgh", 30), ("abcdefgh éß中K", 40)):
        for _ in range(500):
            frm.append("".join(rng.choice(list(alpha), rng.integers(0, hi + 1))))
            to.append("".join(rng.choice(list(alpha), rng.integers(0, hi + 1))))
    # each pair once, via the matrix of one from-string against its partner (and the pair swapped: OSA is symmetric)
    for a, b in zip(frm, to):
        d = osa_oracle.osa_matrix([a, b], [b, a])
        want = osa_py(a, b)
        assert d[0, 0] == want and d[1, 1] == want, (a, b)
    # a swapped copy scores 1 under OSA and 2 under Levenshtein
    d = osa_oracle.osa_matrix(["Jhon", "Micorsoft", "Smtih"], ["John", "Microsoft", "Smith"])
    assert np.diag(d).tolist() == [1, 1, 1]
    assert np.diag(native.editdist_matrix(["Jhon", "Micorsoft", "Smtih"], ["John", "Microsoft", "Smith"], "lev")).tolist() == [2, 2, 2]


def test_oracle_argbest_cutoff_self_and_raw_distance():
    frm = ["Jhon Smtih", "abc", ""]
    to = ["Joan Smyth", "John Smith", "abc", "bac"]
    bi, bs, bd = osa_oracle.osa_argbest(frm, to, "norm_osa")
    assert bi.tolist() == [1, 2, 0] and bs[0] == 0.8 and bd.tolist()[:2] == [2, 0]
    bi, bs, bd = osa_oracle.osa_argbest(frm, to, "norm_osa", score_cutoff=0.9)
    assert bi.tolist() == [-1, 2, -1] and bs.tolist() == [0.0, 1.0, 0.0]
    bi, bs, bd = osa_oracle.osa_argbest(frm, to, "osa", score_cutoff=0.9)      # raw distance: no cutoff, smallest wins
    assert bi.tolist() == [1, 2, 2] and bs.tolist() == [-2.0, -0.0, -3.0] and bd.tolist() == [2, 0, 3]
    s = ["abc", "abc", "bac"]
    bi, _, bd = osa_oracle.osa_argbest(s, s, "osa", exclude_self=True)
    assert bi.tolist() == [1, 0, 0] and bd.tolist() == [0, 0, 1]
    # Levenshtein ties the two candidates at 0.6 and picks the first
    bi, bs, _ = native.editdist_argbest(["Jhon Smtih"], ["Joan Smyth", "John Smith"], "norm_lev")
    assert bi.tolist() == [0] and bs[0] == 0.6


def test_scorer_resolution():
    import types
    from polyfuzz_b200.matchers._rapidfuzz import _resolve_scorer
    from polyfuzz_b200 import EditDistance, RapidFuzz

    def stand_in(name, module):                     # stand-ins with rapidfuzz's function names and module paths
        f = lambda a, b: 0.0                        # noqa: E731
        f.__name__, f.__module__ = name, module
        return f

    for name in ("osa", "OSA", "optimal_string_alignment", "osa_normalized_similarity"):
        assert _resolve_scorer(name, "ratio") == "norm_osa"
        assert EditDistance(scorer=name)._metric == "norm_osa" and RapidFuzz(scorer=name)._metric == "norm_osa"
    for module in ("rapidfuzz.distance.OSA", "rapidfuzz.distance.osa", "rapidfuzz.distance.OSA_py",
                   "rapidfuzz.distance.OSA_cpp", "OSA"):
        f = stand_in("normalized_similarity", module)
        assert EditDistance(scorer=f)._metric == "norm_osa" and RapidFuzz(scorer=f)._metric == "norm_osa", module
    assert RapidFuzz(scorer=stand_in("osa_normalized_similarity", "somewhere"))._metric == "norm_osa"
    # every other normalized_similarity keeps meaning normalised Levenshtein
    for module in ("rapidfuzz.distance.Levenshtein", "rapidfuzz.distance.Levenshtein_cpp", "mypkg.osaka", "mypkg.nosa",
                   "rapidfuzz.distance.DamerauLevenshtein", None):
        f = stand_in("normalized_similarity", module)
        assert EditDistance(scorer=f)._metric == "norm_lev" and RapidFuzz(scorer=f)._metric == "norm_lev", module
    assert EditDistance(scorer="normalized_similarity")._metric == "norm_lev"
    ns = types.SimpleNamespace(__name__="normalized_similarity")        # any object with that __name__
    assert _resolve_scorer(ns, "ratio") == "norm_lev"
    # existing names keep their meaning
    assert EditDistance(scorer="levenshtein")._metric == "norm_lev" and EditDistance()._metric == "ratio"
    assert RapidFuzz()._metric == "WRatio" and RapidFuzz(scorer="ratio")._metric == "ratio"
    with pytest.raises(NotImplementedError, match="'osa'"):
        EditDistance(scorer="damerau_levenshtein")


# ---- host logic with the kernels stubbed ---------------------------------------------------------------------------------
def _rank(frm, to, k, metric, cutoff, exclude_self):
    S = np.array([[osa_oracle.norm_osa(a, b) for b in to] for a in frm])
    oi = np.full((len(frm), k), -1, np.int32); ov = np.zeros((len(frm), k))
    for i in range(len(frm)):
        c = np.array([j for j in range(len(to)) if S[i, j] >= cutoff and not (exclude_self and j == i)], dtype=np.int64)
        if len(c):
            c = c[np.lexsort((c, -S[i, c]))][:k]
            oi[i, :len(c)] = c; ov[i, :len(c)] = S[i, c]
    return oi, ov


@pytest.fixture
def calls(monkeypatch):
    from polyfuzz_b200 import editdist
    seen = []

    def edit_argbest(frm, to, metric="ratio", score_cutoff=0.0, exclude_self=False, **kw):
        seen.append(("edit_argbest", metric, float(score_cutoff), 1))
        i, v = _rank(frm, to, 1, metric, score_cutoff, exclude_self)
        return torch.from_numpy(i[:, 0].copy()), torch.from_numpy(v[:, 0].copy()), torch.zeros(len(frm), dtype=torch.int32)

    def edit_topk(frm, to, k, metric="ratio", score_cutoff=0.0, exclude_self=False, **kw):
        seen.append(("edit_topk", metric, float(score_cutoff), k))
        i, v = _rank(frm, to, k, metric, score_cutoff, exclude_self)
        return torch.from_numpy(i), torch.from_numpy(v)

    monkeypatch.setattr(editdist, "edit_argbest", edit_argbest)
    monkeypatch.setattr(editdist, "edit_topk", edit_topk)
    return seen


def test_rapidfuzz_scale_and_cutoff(calls):
    from polyfuzz_b200 import RapidFuzz
    frm = ["Jhon Smtih", "abcd", "zzzz"]
    to = ["Joan Smyth", "John Smith", "abdc", "abcx"]
    df = RapidFuzz(scorer="osa", score_cutoff=0.7).match(frm, to)
    assert calls == [("edit_argbest", "norm_osa", 0.7, 1)]                 # cutoff on 0..1, like norm_lev
    assert df.To.tolist() == ["John Smith", "abdc", None] and df.Similarity.tolist() == [0.8, 0.75, 0.0]   # not divided by 100
    calls.clear()
    df = RapidFuzz(scorer="osa", score_cutoff=0.7, top_n=3).match(frm, to)
    assert calls == [("edit_topk", "norm_osa", 0.7, 3)]
    assert df.To_2.tolist() == [None, "abcx", None] and df.Similarity_2.tolist() == [0.0, 0.75, 0.0]


def test_editdistance_raw_scores_and_top_n(calls):
    from polyfuzz_b200 import EditDistance
    frm = ["Jhon Smtih", "abcd"]
    to = ["Joan Smyth", "John Smith", "abdc"]
    df = EditDistance(scorer="osa", normalize=False).match(frm, to)
    assert calls[-1] == ("edit_argbest", "norm_osa", float("-inf"), 1)
    assert df.To.tolist() == ["John Smith", "abdc"] and df.Similarity.tolist() == [0.8, 0.75]
    df = EditDistance(scorer="optimal_string_alignment").match(frm, to)              # min-max normalised
    assert df.Similarity.tolist() == [1.0, 0.0]
    df = EditDistance(scorer="osa", normalize=False, top_n=2).match(frm, to)
    assert calls[-1] == ("edit_topk", "norm_osa", float("-inf"), 2)
    assert df.To_2.tolist() == ["Joan Smyth", "Joan Smyth"] and df.Similarity_2.tolist() == [0.6, 1.0 - 9 / 10]   # "a" is shared


def test_metric_ids():
    from polyfuzz_b200 import editdist
    assert editdist.METRIC["osa"] == 6 and editdist.METRIC["norm_osa"] == 7 and "norm_osa" in editdist.TOPK_METRICS
    assert "osa" not in editdist.TOPK_METRICS
    with pytest.raises(ValueError, match="top-k"):
        editdist.edit_topk_staged(None, None, 3, "osa")
