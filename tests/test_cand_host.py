"""Host tests of candidate mode (RapidFuzz / EditDistance with candidates=TFIDF(...)): the constructors' checks, and the frame
assembly for rows without a candidate and for EditDistance's `normalize` over the filled cells.  The device scoring is replaced
by fixed arrays here; tests/test_gpu_cand.py runs it."""
import pickle

import numpy as np
import pandas as pd
import pytest

from polyfuzz_b200 import TFIDF, EditDistance, RapidFuzz
from polyfuzz_b200.matchers import _rapidfuzz

FROM = ["apple", "apples", "pear", "zzz"]
TO = ["apple", "apples", "pears", "mouse"]


@pytest.mark.parametrize("M", [RapidFuzz, EditDistance])
def test_constructor_checks(M):
    for bad in ("tfidf", 3, object(), RapidFuzz()):
        with pytest.raises(ValueError, match="TFIDF"):
            M(candidates=bad)
    with pytest.raises(ValueError, match="exceeds the candidates' top_n"):
        M(top_n=4, candidates=TFIDF(top_n=3))
    with pytest.raises(ValueError, match="distributed"):
        M(distributed=True, candidates=TFIDF(top_n=3))
    # accepted: top_n up to the TF-IDF's, and a distributed TF-IDF
    assert M(top_n=3, candidates=TFIDF(top_n=3)).candidates.top_n == 3
    assert M(candidates=TFIDF(top_n=10, distributed=True)).candidates.distributed
    assert M().candidates is None
    # the top_n check still comes first
    with pytest.raises(ValueError, match="1 to 32"):
        M(top_n=33, candidates=TFIDF(top_n=40))


def test_pickle_keeps_the_candidate_source():
    m = RapidFuzz(top_n=2, candidates=TFIDF(top_n=5, min_similarity=0))
    r = pickle.loads(pickle.dumps(m))
    assert isinstance(r.candidates, TFIDF) and r.candidates.top_n == 5 and r.candidates.min_similarity == 0


def _fixed(monkeypatch, idx, score):
    """Make the candidate scoring return fixed host arrays; records the calls."""
    calls = []

    def fake(from_list, targets, metric, cutoff, self_match, k, candidates, to_list, re_train, kept):
        calls.append(dict(metric=metric, cutoff=cutoff, self_match=self_match, k=k, re_train=re_train))
        return np.asarray(idx, np.int32)[:, :k], np.asarray(score, np.float64)[:, :k]
    monkeypatch.setattr(_rapidfuzz, "_cand_topk", fake)
    return calls


def test_rapidfuzz_frame_with_empty_rows(monkeypatch):
    calls = _fixed(monkeypatch, [[1, 0], [-1, -1], [2, -1], [-1, -1]], [[90.0, 80.0], [0.0, 0.0], [50.0, 0.0], [0.0, 0.0]])
    got = RapidFuzz(top_n=2, score_cutoff=0.3, candidates=TFIDF(top_n=3)).match(FROM, TO)
    assert calls[0]["metric"] == "WRatio" and calls[0]["cutoff"] == 30.0 and calls[0]["k"] == 2 and not calls[0]["self_match"]
    assert list(got.columns) == ["From", "To", "Similarity", "To_2", "Similarity_2"]
    assert got.To.tolist() == ["apples", None, "pears", None] and got.To_2.tolist() == ["apple", None, None, None]
    assert got.Similarity.tolist() == [0.9, 0.0, 0.5, 0.0] and got.Similarity_2.tolist() == [0.8, 0.0, 0.0, 0.0]
    # top_n = 1: the columns of the all-pairs frame
    _fixed(monkeypatch, [[1], [-1], [2], [-1]], [[90.0], [0.0], [50.0], [0.0]])
    one = RapidFuzz(candidates=TFIDF(top_n=3)).match(FROM, TO, re_train=False)
    exp = pd.DataFrame({"From": pd.Series(FROM, dtype=object), "To": pd.Series(["apples", None, "pears", None], dtype=object),
                        "Similarity": [0.9, 0.0, 0.5, 0.0]})
    pd.testing.assert_frame_equal(one, exp)


def test_editdistance_empty_rows_and_normalize(monkeypatch):
    idx = [[1, 0], [-1, -1], [2, -1], [3, 1]]
    score = [[0.9, 0.8], [0.0, 0.0], [0.5, 0.0], [0.2, 0.1]]
    calls = _fixed(monkeypatch, idx, score)
    raw = EditDistance(scorer="levenshtein", top_n=2, normalize=False, candidates=TFIDF(top_n=2)).match(FROM, TO)
    assert calls[0]["metric"] == "norm_lev" and calls[0]["cutoff"] == float("-inf")
    assert raw.To.tolist() == ["apples", None, "pears", "mouse"] and raw.Similarity.tolist() == [0.9, 0.0, 0.5, 0.2]
    norm = EditDistance(scorer="levenshtein", top_n=2, candidates=TFIDF(top_n=2)).match(FROM, TO)
    # one min and one max over the filled cells (0.1 .. 0.9); empty slots stay (None, 0.0)
    filled = np.array(idx) >= 0
    s = np.array(score)
    exp = np.where(filled, (s - 0.1) / (0.9 - 0.1), 0.0)
    np.testing.assert_array_equal(norm[["Similarity", "Similarity_2"]].to_numpy(), exp)
    assert norm.To_2.tolist() == ["apple", None, None, "apples"]
    # top_n = 1 with an empty row: (None, 0.0), normalised over the filled rows
    _fixed(monkeypatch, [[1], [-1], [2], [3]], [[90.0], [0.0], [50.0], [10.0]])
    one = EditDistance(candidates=TFIDF(top_n=2)).match(FROM, TO)
    assert list(one.columns) == ["From", "To", "Similarity"]
    assert one.To.tolist() == ["apples", None, "pears", "mouse"]
    np.testing.assert_array_equal(one.Similarity.to_numpy(), [1.0, 0.0, 0.5, 0.0])
    # no filled cell at all: every slot (None, 0.0)
    _fixed(monkeypatch, [[-1]] * 4, [[0.0]] * 4)
    none = EditDistance(candidates=TFIDF(top_n=2)).match(FROM, TO)
    assert none.To.isna().all() and (none.Similarity == 0.0).all()


def test_self_match_is_passed_on(monkeypatch):
    calls = _fixed(monkeypatch, [[1], [0], [-1], [-1]], [[90.0], [90.0], [0.0], [0.0]])
    got = RapidFuzz(scorer="ratio", candidates=TFIDF(top_n=3)).match(FROM)
    assert calls[0]["self_match"] and calls[0]["metric"] == "ratio"
    assert got.To.tolist() == ["apples", "apple", None, None]
