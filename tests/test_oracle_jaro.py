"""CPU tests of the Jaro / Jaro-Winkler oracle (tests/jaro_oracle.c) and of the scorer names the matchers accept.
The oracle is pinned on published known answers (tests/golden/jaro_published.json, sources inside) and on a literal
Python transcription of the definition."""
import json
import os

import numpy as np
import pytest

import jaro_oracle


@pytest.fixture(scope="module")
def published(golden_dir):
    return json.load(open(os.path.join(golden_dir, "jaro_published.json")))


def _jaro_py(s1, s2, winkler):
    """The definition step by step (jellyfish's jaro_similarity / jaro_winkler_similarity, long_tolerance=False)."""
    l1, l2 = len(s1), len(s2)
    if not l1 or not l2:
        return 0.0, 0
    r = max(0, max(l1, l2) // 2 - 1)
    f1, f2 = [False] * l1, [False] * l2
    m = 0
    for i, c in enumerate(s1):
        for j in range(max(0, i - r), min(i + r, l2 - 1) + 1):
            if not f2[j] and s2[j] == c:
                f1[i] = f2[j] = True
                m += 1
                break
    if not m:
        return 0.0, 0
    p1 = [s1[i] for i in range(l1) if f1[i]]
    p2 = [s2[j] for j in range(l2) if f2[j]]
    t = sum(a != b for a, b in zip(p1, p2)) // 2
    mf = float(m)
    jaro = (mf / l1 + mf / l2 + (mf - t) / mf) / 3
    if winkler and jaro > 0.7:
        p = 0
        while p < min(l1, l2, 4) and s1[p] == s2[p]:
            p += 1
        if p:
            jaro = jaro + (p * 0.1) * (1.0 - jaro)
    return jaro, m


def test_published_vectors(published):
    assert len(published["pairs"]) >= 7
    for v in published["pairs"]:
        got, m = jaro_oracle.jaro_pair(v["a"], v["b"], winkler=v["fn"] == "jaro_winkler_similarity")
        if v["digits"] is None:
            assert got == v["expect"], (v, got)
        else:
            assert round(got, v["digits"]) == v["expect"], (v, got)
        assert got == _jaro_py(v["a"], v["b"], v["fn"] == "jaro_winkler_similarity")[0]
    # the full doubles of the Wikipedia pairs (same restatement)
    assert jaro_oracle.jaro_pair("MARTHA", "MARHTA") == (0.9611111111111111, 6)
    assert jaro_oracle.jaro_pair("DWAYNE", "DUANE") == (0.8400000000000001, 4)
    assert jaro_oracle.jaro_pair("DIXON", "DICKSONX") == (0.8133333333333332, 4)


def test_oracle_equals_definition_on_random_pairs():
    rng = np.random.default_rng(5)
    for alpha, hi in (("ab", 12), ("abc", 12), ("abcdefgh éß中", 40)):
        for _ in range(1500):
            a = "".join(rng.choice(list(alpha), rng.integers(0, hi + 1)))
            b = "".join(rng.choice(list(alpha), rng.integers(0, hi + 1)))
            for w in (False, True):
                assert jaro_oracle.jaro_pair(a, b, w) == _jaro_py(a, b, w), (a, b, w)
    assert jaro_oracle.jaro_pair("", "abc") == (0.0, 0) and jaro_oracle.jaro_pair("abc", "") == (0.0, 0)
    assert jaro_oracle.jaro_pair("abc", "xyz") == (0.0, 0)


def test_oracle_argbest_first_maximum_cutoff_and_self():
    frm = ["martha", "dwayne", "dixon", ""]
    to = ["marhta", "martha", "duane", "dickson", "martha"]
    bi, bs, bd = jaro_oracle.jaro_argbest(frm, to, "jaro_winkler")
    assert bi.tolist() == [1, 2, 3, 0] and bs[0] == 1.0 and bd.tolist()[:3] == [6, 4, 4] and bs[3] == 0.0
    bi, bs, bd = jaro_oracle.jaro_argbest(frm, to, "jaro", score_cutoff=0.9)
    assert bi.tolist() == [1, -1, -1, -1] and bd.tolist() == [6, -1, -1, -1] and bs.tolist()[1:] == [0.0, 0.0, 0.0]
    s = ["dup", "dup", "other"]
    bi, _, _ = jaro_oracle.jaro_argbest(s, s, "jaro_winkler", exclude_self=True)
    assert bi.tolist()[:2] == [1, 0]


def test_scorer_resolution():
    from polyfuzz_b200.matchers._rapidfuzz import _resolve_scorer
    from polyfuzz_b200 import EditDistance, RapidFuzz

    def jaro_similarity(a, b):                      # stand-ins with jellyfish's function names
        return 0.0

    def jaro_winkler_similarity(a, b):
        return 0.0

    assert _resolve_scorer(jaro_winkler_similarity, "ratio", allow_jaro=True) == "jaro_winkler"
    assert _resolve_scorer(jaro_similarity, "ratio", allow_jaro=True) == "jaro"
    for name, want in (("jaro", "jaro"), ("jaro_similarity", "jaro"), ("jaro_winkler", "jaro_winkler"),
                       ("jaro_winkler_similarity", "jaro_winkler")):
        assert _resolve_scorer(name, "ratio", allow_jaro=True) == want
        assert EditDistance(scorer=name)._metric == want
    assert EditDistance(n_jobs=1, scorer=jaro_winkler_similarity)._metric == "jaro_winkler"
    assert EditDistance(scorer=jaro_similarity)._metric == "jaro"
    for sc in (jaro_winkler_similarity, jaro_similarity, "jaro_winkler", "jaro"):
        with pytest.raises(NotImplementedError):
            RapidFuzz(scorer=sc)
    # every existing name keeps its meaning
    assert EditDistance(scorer="normalized_similarity")._metric == "norm_lev"
    assert EditDistance(scorer="ratio")._metric == "ratio" and EditDistance()._metric == "ratio"
    assert RapidFuzz(scorer="ratio")._metric == "ratio" and RapidFuzz()._metric == "WRatio"
    with pytest.raises(NotImplementedError):
        EditDistance(scorer=lambda a, b: 1.0)
