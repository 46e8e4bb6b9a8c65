"""CPU tests of the unrestricted Damerau-Levenshtein (DL) metrics: the oracle's full-matrix Lowrance-Wagner DP
(tests/dl_oracle.c) against a literal Python transcription and known values, the bounds that gate the GPU kernel
(max(ceil(lev/2), ceil(2*osa/3), ||a|-|b||) <= dl <= osa), the scorer names that resolve to DL, and the matchers' host logic
with the kernels stubbed."""
import numpy as np
import pytest
import torch

import dl_oracle
import osa_oracle
from oracle import native

dl = dl_oracle.dl


def dl_py(a, b):
    """Lowrance-Wagner with unit costs: the full (|a|+2) x (|b|+2) matrix and a dict of the last row of each character."""
    la, lb = len(a), len(b)
    inf = la + lb
    d = [[0] * (lb + 2) for _ in range(la + 2)]
    d[0][0] = inf
    for i in range(la + 1):
        d[i + 1][0], d[i + 1][1] = inf, i
    for j in range(lb + 1):
        d[0][j + 1], d[1][j + 1] = inf, j
    last_row = {}
    for i in range(1, la + 1):
        last_col = 0
        for j in range(1, lb + 1):
            k, l = last_row.get(b[j - 1], 0), last_col
            cost = 0 if a[i - 1] == b[j - 1] else 1
            if cost == 0:
                last_col = j
            d[i + 1][j + 1] = min(d[i][j] + cost, d[i + 1][j] + 1, d[i][j + 1] + 1, d[k][l] + (i - k - 1) + 1 + (j - l - 1))
        last_row[a[i - 1]] = i
    return d[la + 1][lb + 1]


def _random_pairs(seed, n_each):
    rng = np.random.default_rng(seed)
    frm, to = [], []
    for alpha, hi in (("ab", 10), ("abc", 14), ("abcd", 16), ("abcdefgh", 30), ("abcdefgh éß中K", 40)):
        for _ in range(n_each):
            frm.append("".join(rng.choice(list(alpha), rng.integers(0, hi + 1))))
            to.append("".join(rng.choice(list(alpha), rng.integers(0, hi + 1))))
    return frm, to


def test_known_values():
    assert dl("CA", "ABC") == 2 and osa_oracle.osa("CA", "ABC") == 3
    assert dl("abc", "ca") == 2 and osa_oracle.osa("abc", "ca") == 3
    assert dl("jellyfish", "jellyfihs") == 1
    assert dl("", "abc") == 3 and dl("abc", "") == 3 and dl("", "") == 0
    assert dl("ab", "ba") == 1 and dl("kitten", "sitting") == 3
    for a, b in (("CA", "ABC"), ("abc", "ca"), ("jellyfish", "jellyfihs"), ("", "abc"), ("abcdef", "badcfe")):
        assert dl(a, b) == dl(b, a) == dl_py(a, b)
    # DL is a metric where OSA is not: osa(CA, AC) + osa(AC, ABC) = 2 < osa(CA, ABC) = 3
    assert dl("CA", "AC") + dl("AC", "ABC") >= dl("CA", "ABC")
    _, bs, bd = dl_oracle.dl_argbest(["CA"], ["ABC"], "norm_dl")
    assert bs[0] == 1.0 - 2 / 3 and bd[0] == 2
    _, bs, _ = dl_oracle.dl_argbest([""], [""], "norm_dl")
    assert bs[0] == 1.0


def test_oracle_equals_definition_on_random_pairs():
    frm, to = _random_pairs(5, 450)
    assert len(frm) >= 2000
    for a, b in zip(frm, to):
        d = dl_oracle.dl_matrix([a, b], [b, a])
        want = dl_py(a, b)
        assert d[0, 0] == want and d[1, 1] == want, (a, b)


def test_bounds_that_gate_the_kernel():
    """max(ceil(lev/2), ceil(2*osa/3), ||a|-|b||) <= dl <= osa <= lev on random pairs over small alphabets; ("CA", "ABC")
    reaches osa = 1.5 * dl."""
    frm, to = _random_pairs(17, 1000)
    d = np.array([dl_oracle.dl_matrix([a], [b])[0, 0] for a, b in zip(frm, to)])
    o = np.array([osa_oracle.osa_matrix([a], [b])[0, 0] for a, b in zip(frm, to)])
    lev = np.array([int(native.editdist_matrix([a], [b], "lev")[0, 0]) for a, b in zip(frm, to)])
    dlen = np.abs(np.array([len(a) - len(b) for a, b in zip(frm, to)]))
    lower = np.maximum(np.maximum((lev + 1) // 2, (2 * o + 2) // 3), dlen)
    assert (lower <= d).all() and (d <= o).all() and (o <= lev).all()
    assert ((2 * o + 2) // 3 == d).any() and (d < o).any()
    assert 2 * osa_oracle.osa("CA", "ABC") == 3 * dl("CA", "ABC")


def test_oracle_argbest_cutoff_self_and_raw_distance():
    frm = ["CA", "abc", ""]
    to = ["XY", "ABC", "abc", "bca"]
    bi, bs, bd = dl_oracle.dl_argbest(frm, to, "norm_dl")
    assert bi.tolist() == [1, 2, 0] and bs[0] == 1.0 - 2 / 3 and bd.tolist() == [2, 0, 2]
    bi, bs, _ = dl_oracle.dl_argbest(frm, to, "norm_dl", score_cutoff=0.5)
    assert bi.tolist() == [-1, 2, -1] and bs.tolist() == [0.0, 1.0, 0.0]
    bi, bs, bd = dl_oracle.dl_argbest(frm, to, "dl", score_cutoff=0.9)       # raw distance: no cutoff, smallest wins
    assert bi.tolist() == [0, 2, 0] and bs.tolist() == [-2.0, -0.0, -2.0] and bd.tolist() == [2, 0, 2]
    s = ["abc", "abc", "bac"]
    bi, _, bd = dl_oracle.dl_argbest(s, s, "dl", exclude_self=True)
    assert bi.tolist() == [1, 0, 0] and bd.tolist() == [0, 0, 1]


def _stand_in(name, module):                        # stand-ins with rapidfuzz's function names and module paths
    f = lambda a, b: 0.0                            # noqa: E731
    f.__name__, f.__module__ = name, module
    return f


def test_scorer_resolution():
    from polyfuzz_b200.matchers._rapidfuzz import _resolve_scorer
    from polyfuzz_b200 import EditDistance, RapidFuzz
    for name in ("dl", "DL", "unrestricted_damerau_levenshtein", "Unrestricted_Damerau_Levenshtein",
                 "damerau_levenshtein_normalized_similarity"):
        assert _resolve_scorer(name, "ratio") == "norm_dl"
        assert EditDistance(scorer=name)._metric == "norm_dl" and RapidFuzz(scorer=name)._metric == "norm_dl"
        f = _stand_in(name, "somewhere")
        assert EditDistance(scorer=f)._metric == "norm_dl" and RapidFuzz(scorer=f)._metric == "norm_dl"
    # the bare name stays ambiguous, and the message names both choices
    for cls in (EditDistance, RapidFuzz):
        with pytest.raises(NotImplementedError, match="'osa'") as e:
            cls(scorer="damerau_levenshtein")
        assert "'dl'" in str(e.value)
    # DamerauLevenshtein.normalized_similarity keeps resolving to normalised Levenshtein (a separate fix)
    f = _stand_in("normalized_similarity", "rapidfuzz.distance.DamerauLevenshtein")
    assert EditDistance(scorer=f)._metric == "norm_lev" and RapidFuzz(scorer=f)._metric == "norm_lev"
    assert EditDistance(scorer="osa")._metric == "norm_osa" and EditDistance()._metric == "ratio"


def test_metric_ids():
    from polyfuzz_b200 import editdist
    assert editdist.METRIC["dl"] == 8 and editdist.METRIC["norm_dl"] == 9
    assert "norm_dl" in editdist.TOPK_METRICS and "dl" not in editdist.TOPK_METRICS
    with pytest.raises(ValueError, match="top-k"):
        editdist.edit_topk_staged(None, None, 3, "dl")


# ---- host logic with the kernels stubbed ---------------------------------------------------------------------------------
def _rank(frm, to, k, cutoff, exclude_self):
    S = np.array([[dl_oracle.norm_dl(a, b) for b in to] for a in frm])
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
        i, v = _rank(frm, to, 1, score_cutoff, exclude_self)
        return torch.from_numpy(i[:, 0].copy()), torch.from_numpy(v[:, 0].copy()), torch.zeros(len(frm), dtype=torch.int32)

    def edit_topk(frm, to, k, metric="ratio", score_cutoff=0.0, exclude_self=False, **kw):
        seen.append(("edit_topk", metric, float(score_cutoff), k))
        i, v = _rank(frm, to, k, score_cutoff, exclude_self)
        return torch.from_numpy(i), torch.from_numpy(v)

    monkeypatch.setattr(editdist, "edit_argbest", edit_argbest)
    monkeypatch.setattr(editdist, "edit_topk", edit_topk)
    return seen


def test_editdistance_issue_example(calls):
    from polyfuzz_b200 import EditDistance
    df = EditDistance(scorer="dl", normalize=False).match(["CA"], ["ABC", "XY"])
    assert calls == [("edit_argbest", "norm_dl", float("-inf"), 1)]
    assert df.To.tolist() == ["ABC"] and df.Similarity.tolist() == [1.0 - 2 / 3]
    df = EditDistance(scorer="dl", normalize=False, top_n=2).match(["CA", "abc"], ["ABC", "XY", "bca"])
    assert calls[-1] == ("edit_topk", "norm_dl", float("-inf"), 2)
    assert df.To.tolist() == ["ABC", "bca"] and df.To_2.tolist() == ["XY", "ABC"]


def test_rapidfuzz_scale_and_cutoff(calls):
    from polyfuzz_b200 import RapidFuzz
    frm = ["CA", "abcd", "zzzz"]
    to = ["ABC", "XY", "abdc", "abcx"]
    df = RapidFuzz(scorer="dl", score_cutoff=0.3).match(frm, to)
    assert calls == [("edit_argbest", "norm_dl", 0.3, 1)]                  # cutoff on 0..1, like norm_lev
    assert df.To.tolist() == ["ABC", "abdc", None] and df.Similarity.tolist() == [1.0 - 2 / 3, 0.75, 0.0]   # not divided by 100
    calls.clear()
    df = RapidFuzz(scorer="unrestricted_damerau_levenshtein", score_cutoff=0.7, top_n=3).match(frm, to)
    assert calls == [("edit_topk", "norm_dl", 0.7, 3)]
    assert df.To_2.tolist() == [None, "abcx", None] and df.Similarity_2.tolist() == [0.0, 0.75, 0.0]
