"""Indel, LCSseq, Hamming, Prefix and Postfix, CPU only: the plain-Python oracle (tests/seq_oracle.py) on hand-computed values and
against independent restatements (fuzz.ratio's ns, the C LCS, os.path.commonprefix), the scorer names of the matchers, the argument
rules of pfz_lev_rows for metrics 10..16, and the matchers' host logic with the kernels stubbed."""
import ctypes
import functools
import itertools
import os
import pickle

import numpy as np
import pytest
import torch

import seq_oracle
from seq_oracle import METRICS, similarity

NAMES = {"norm_indel": ("indel", "indel_normalized_similarity"),
         "norm_lcsseq": ("lcsseq", "lcs_seq", "lcsseq_normalized_similarity", "lcs_seq_normalized_similarity"),
         "norm_hamming": ("hamming", "hamming_normalized_similarity"),
         "norm_prefix": ("prefix", "prefix_normalized_similarity"),
         "norm_postfix": ("postfix", "postfix_normalized_similarity")}


def _rand_pairs(seed, n, alpha, hi=12):
    rng = np.random.default_rng(seed)
    s = lambda: "".join(alpha[i] for i in rng.integers(0, len(alpha), rng.integers(0, hi + 1)))   # noqa: E731
    return [(s(), s()) for _ in range(n)]


# ---- the oracle ------------------------------------------------------------------------------------------------------------
KNOWN = [
    # (a, b, {metric: score}) -- worked by hand from the definitions
    ("", "", {m: 1.0 for m in METRICS}),
    ("abc", "", {m: 0.0 for m in METRICS}),
    ("", "xy", {m: 0.0 for m in METRICS}),
    # LCS("kitten", "sitting") = 4 ("ittn"); Hamming: k/s and e/i differ, plus 1 surplus; no common prefix or suffix
    ("kitten", "sitting", {"norm_indel": 1 - 5 / 13, "norm_lcsseq": 1 - 3 / 7, "norm_hamming": 1 - 3 / 7, "norm_prefix": 0.0,
                           "norm_postfix": 0.0}),
    ("abcde", "abxde", {"norm_indel": 0.8, "norm_lcsseq": 0.8, "norm_hamming": 0.8, "norm_prefix": 0.4, "norm_postfix": 0.4}),
    ("abcd", "ab", {"norm_indel": 1 - 2 / 6, "norm_lcsseq": 0.5, "norm_hamming": 0.5, "norm_prefix": 0.5, "norm_postfix": 0.0}),
    ("xyab", "ab", {"norm_indel": 1 - 2 / 6, "norm_lcsseq": 0.5, "norm_hamming": 0.0, "norm_prefix": 0.0, "norm_postfix": 0.5}),
    ("same", "same", {m: 1.0 for m in METRICS}),
    # non-ASCII and astral code points count as one symbol each
    ("é中😀a", "é中😀b", {"norm_indel": 0.75, "norm_lcsseq": 0.75, "norm_hamming": 0.75, "norm_prefix": 0.75, "norm_postfix": 0.0}),
    ("😀x", "y😀x", {"norm_indel": 0.8, "norm_lcsseq": 1 - 1 / 3, "norm_hamming": 0.0, "norm_prefix": 0.0, "norm_postfix": 1 - 1 / 3}),
    ("Intl Business Machines", "International Business Machines",
     # LCS = 22 (all of the short one); 6 of the first 22 positions agree; prefix "Int", suffix "l Business Machines"
     {"norm_indel": 1 - 9 / 53, "norm_lcsseq": 1 - 9 / 31, "norm_hamming": 1 - 25 / 31, "norm_prefix": 1 - 28 / 31,
      "norm_postfix": 1 - 12 / 31}),
]


@pytest.mark.parametrize("a,b,want", KNOWN)
def test_known_values(a, b, want):
    for metric, v in want.items():
        assert similarity(metric, a, b) == v, (metric, a, b)


def test_symmetric_metrics_and_bounds():
    for a, b in _rand_pairs(1, 400, "abé中😀"):
        for metric in METRICS:
            d, mx = seq_oracle.dist_max(metric, a, b)
            assert 0 <= d <= mx and 0.0 <= similarity(metric, a, b) <= 1.0
            assert seq_oracle.dist_max(metric, b, a) == (d, mx)
            assert (d == 0) == (a == b) or metric in ("norm_indel", "norm_lcsseq") or mx == 0


def test_indel_is_ratio_ns():
    """Indel's score is fuzz.ratio's ns (before the x100) as a double, and differs from ratio / 100 where the round trip does."""
    from oracle import fuzz
    for a, b in _rand_pairs(2, 600, "abcd中"):
        assert similarity("norm_indel", a, b) == fuzz._indel_norm_sim(a, b)
    a, b = "aaaaab", "aaaaac"                           # indel 2 of 12: ns = 1 - 2/12, and (ns * 100) / 100 != ns
    ns = similarity("norm_indel", a, b)
    assert ns == 1 - 2 / 12 and fuzz.ratio(a, b) / 100 != ns


def test_lcs_agrees_with_the_c_oracle():
    import lcs_oracle
    pairs = _rand_pairs(3, 300, "ab中😀", hi=40) + [("a" * 300, "ba" * 200), ("", "abc")]
    for a, b in pairs:
        assert seq_oracle.lcs_len(a, b) == lcs_oracle.lcs_len(a, b)
    frm = [p[0] for p in pairs[:25]]; to = [p[1] for p in pairs[25:60]]
    np.testing.assert_array_equal(seq_oracle.lcs_matrix(frm, to, fast=True), seq_oracle.lcs_matrix(frm, to, fast=False))


def test_positional_identities():
    for a, b in _rand_pairs(4, 600, "ab中"):
        assert seq_oracle.common_prefix(a, b) == len(os.path.commonprefix([a, b]))
        assert seq_oracle.common_suffix(a, b) == len(os.path.commonprefix([a[::-1], b[::-1]]))
        if len(a) == len(b):                           # equal lengths: the plain Hamming distance over n
            d = sum(x != y for x, y in zip(a, b))
            assert similarity("norm_hamming", a, b) == (1.0 - d / len(a) if a else 1.0)
        else:                                          # pad=True: the surplus counts as mismatches, as padding would
            short, long_ = sorted((a, b), key=len)
            padded = short + "\uffff" * (len(long_) - len(short))
            assert seq_oracle.dist_max("norm_hamming", a, b)[0] == sum(x != y for x, y in zip(padded, long_))


def test_topk_key_and_cutoff():
    frm, to = ["abc", "abd", ""], ["abd", "abc", "abc", "", "x"]
    D, M, S = seq_oracle.matrices("norm_prefix", frm, to)
    idx, sc, dist = seq_oracle.topk_from(S, D, 3, 0.5)
    assert idx[0].tolist() == [1, 2, 0] and sc[0].tolist() == [1.0, 1.0, 1 - 1 / 3] and dist[0].tolist() == [0, 0, 1]
    assert idx[2].tolist() == [3, -1, -1] and sc[2].tolist() == [1.0, 0.0, 0.0]
    idx, _, _ = seq_oracle.topk_from(S, D, 2, 0.0, exclude_self=True)
    assert idx[1].tolist() == [0, 2]


# ---- scorer names ----------------------------------------------------------------------------------------------------------
def _stand_in(name, module):                        # stand-ins with rapidfuzz's function names and module paths
    f = lambda a, b, **kw: 0.0                      # noqa: E731
    f.__name__, f.__module__ = name, module
    return f


def test_new_names_resolve():
    from polyfuzz_b200 import EditDistance, RapidFuzz
    from polyfuzz_b200.matchers._rapidfuzz import _resolve_scorer
    for metric, names in NAMES.items():
        for name in names:
            for s in (name, name.upper(), _stand_in(name, "rapidfuzz.distance"), _stand_in(name, "somewhere")):
                assert _resolve_scorer(s, "ratio") == metric and _resolve_scorer(s, "WRatio", allow_jaro=True) == metric
            for cls in (EditDistance, RapidFuzz):
                assert cls(scorer=name)._metric == metric
        with pytest.raises(NotImplementedError, match="partial"):
            EditDistance(scorer=functools.partial(_stand_in(names[0], "x"), weights=(1, 1, 2)))


def test_existing_names_keep_their_metric():
    from polyfuzz_b200 import fuzzy
    from polyfuzz_b200.matchers._rapidfuzz import _JARO, _NAMES, _resolve_scorer
    new = {n for names in NAMES.values() for n in names}
    old = {"ratio": "ratio", "levenshtein": "norm_lev", "norm_lev": "norm_lev", "normalized_similarity": "norm_lev",
           "normalized_levenshtein": "norm_lev", "osa": "norm_osa", "optimal_string_alignment": "norm_osa",
           "osa_normalized_similarity": "norm_osa", "dl": "norm_dl", "unrestricted_damerau_levenshtein": "norm_dl",
           "damerau_levenshtein_normalized_similarity": "norm_dl"}
    assert set(_NAMES) == set(old) | new
    for name, metric in old.items():
        assert _resolve_scorer(name, "ratio") == metric and _resolve_scorer(_stand_in(name, "somewhere"), "ratio") == metric
    for name, metric in _JARO.items():
        assert _resolve_scorer(name, "ratio", allow_jaro=True) == metric
    for name in fuzzy.SCORER:
        assert _resolve_scorer(name, "ratio") == name
    with pytest.raises(NotImplementedError, match="ambiguous"):
        _resolve_scorer("damerau_levenshtein", "ratio")
    with pytest.raises(NotImplementedError):
        _resolve_scorer("jaro", "ratio")                # Jaro stays EditDistance-only


def test_normalized_similarity_callables_keep_norm_lev():
    """rapidfuzz.distance.<Module>.normalized_similarity resolves by the existing rule: OSA for OSA modules, normalised
    Levenshtein for every other -- these five included (re-pointing them changes existing results)."""
    from polyfuzz_b200.matchers._rapidfuzz import _resolve_scorer
    for mod in ("Indel", "LCSseq", "Hamming", "Prefix", "Postfix", "DamerauLevenshtein", "Levenshtein"):
        for suffix in ("", "_py", "_cpp"):
            f = _stand_in("normalized_similarity", f"rapidfuzz.distance.{mod}{suffix}")
            assert _resolve_scorer(f, "ratio") == "norm_lev" and _resolve_scorer(f, "WRatio", allow_jaro=True) == "norm_lev"
    assert _resolve_scorer(_stand_in("normalized_similarity", "rapidfuzz.distance.OSA"), "ratio") == "norm_osa"


def test_metric_tables():
    from polyfuzz_b200 import editdist
    assert {m: editdist.METRIC[m] for m in METRICS} == {"norm_indel": 11, "norm_lcsseq": 12, "norm_hamming": 13, "norm_prefix": 14,
                                                        "norm_postfix": 15}
    assert 10 not in editdist.METRIC.values()
    assert all(m in editdist.TOPK_METRICS for m in METRICS)
    for m in METRICS:
        with pytest.raises(ValueError, match="matrix"):
            editdist.edit_argbest_staged(None, None, m, want_matrix=True)


# ---- pfz_lev_rows argument rules for metrics 10..16 (n_ids = 0, null buffers: nothing is read) ---------------------------------
BUF = np.zeros(64, dtype=np.int64)
NN = ctypes.c_void_p(BUF.ctypes.data)
SOURCES = [(None, 1, 0, None), (None, 3, 0, None), (None, 0, 0, None), (NN, 1, 4, NN), (NN, 2, 4, NN), (NN, 1, 0, NN),
           (NN, 1, 4, None)]


def _rules(metric, k, part_dist, matrix, gate, source):
    cand, n_splits, c, pos_of = source
    broken = []
    if cand is not None:
        broken += ["candidate mode"] if n_splits != 1 or c < 1 or pos_of is None else []
    elif n_splits < 1:
        broken.append("n_splits < 1")
    if not 11 <= metric <= 15:
        broken.append("unknown metric")
    if not 0 <= k <= 32:
        broken.append(f"k={k} unsupported")
    if k >= 1 and (part_dist or matrix):
        broken.append("top-k has no distance output")
    if k == 0 and not part_dist:
        broken.append("arg-best needs part_dist")
    if matrix:
        broken.append("distance matrix is not available")
    if gate:
        broken.append("gate is for DL / NORM_DL only")
    return broken


def test_lev_rows_rules_for_the_new_metrics():
    from polyfuzz_b200 import _lib
    lib = _lib.load()
    n_allowed = 0
    for metric, k, part_dist, matrix, gate, source in itertools.product(range(10, 17), (-1, 0, 1, 5, 32, 33), (False, True),
                                                                         (False, True), (False, True), SOURCES):
        cand, n_splits, c, pos_of = source
        rc = lib.pfz_lev_rows(NN, NN, 10, NN, 0, 0, NN, NN, NN, NN, NN, 20, metric, 0.5, 0, 0, n_splits, k, cand, c, pos_of, NN, NN,
                              NN if part_dist else None, NN if matrix else None, 20 if matrix else 0, NN if gate else None, NN, None)
        broken = _rules(metric, k, part_dist, matrix, gate, source)
        msg = lib.pfz_last_error().decode()
        if not broken:
            assert rc == 0, (metric, k, part_dist, matrix, gate, source, msg)
            n_allowed += 1
        else:
            assert rc == 1 and any(b in msg for b in broken), (metric, k, part_dist, matrix, gate, source, broken, msg)
    assert n_allowed == 5 * 4 * 3          # 5 metrics x (arg-best with part_dist + 3 top-k sizes) x 3 valid sources
    for metric in METRICS:                 # every word class is accepted
        for n_words in (0, 1, 2, 4, 8, 16):
            from polyfuzz_b200 import editdist
            rc = lib.pfz_lev_rows(NN, NN, 10, NN, 0, n_words, NN, NN, NN, NN, NN, 20, editdist.METRIC[metric], 0.5, 0, 0, 1, 3, None, 0,
                                  None, NN, NN, None, None, 0, None, NN, None)
            assert rc == 0, lib.pfz_last_error().decode()


# ---- matcher host logic with the kernels stubbed ------------------------------------------------------------------------------
FROM = ["kitten", "Jhon Smtih", "Micorsoft", "apple", "appel", "house", "", "Intl Business Machines"]
TO = ["sitting", "XY", "Joan Smyth", "John Smith", "Microsoft", "apple", "apples", "mouse", "International Business Machines"]


@pytest.fixture
def calls(monkeypatch):
    from polyfuzz_b200 import editdist
    seen = []

    def edit_argbest(frm, to, metric="ratio", score_cutoff=0.0, exclude_self=False, **kw):
        seen.append(("argbest", metric, float(score_cutoff), 1, kw.get("reuse")))
        i, s, d = seq_oracle.argbest(metric, frm, to, score_cutoff, exclude_self)
        return torch.from_numpy(i.copy()), torch.from_numpy(s.copy()), torch.from_numpy(d.astype(np.int32))

    def edit_topk(frm, to, k, metric="ratio", score_cutoff=0.0, exclude_self=False, **kw):
        seen.append(("topk", metric, float(score_cutoff), k, kw.get("reuse")))
        i, s, _ = seq_oracle.topk(metric, frm, to, k, score_cutoff, exclude_self)
        return torch.from_numpy(i), torch.from_numpy(s)

    monkeypatch.setattr(editdist, "edit_argbest", edit_argbest)
    monkeypatch.setattr(editdist, "edit_topk", edit_topk)
    return seen


@pytest.mark.parametrize("name", ["indel", "lcs_seq", "hamming", "prefix", "postfix"])
def test_rapidfuzz_frames(calls, name):
    from polyfuzz_b200 import RapidFuzz
    metric = RapidFuzz(scorer=name)._metric
    df = RapidFuzz(scorer=name, score_cutoff=0.5).match(FROM, TO)
    assert calls == [("argbest", metric, 0.5, 1, False)]                 # the cutoff on 0..1
    oi, os_, _ = seq_oracle.argbest(metric, FROM, TO, 0.5)
    assert df.To.tolist() == [TO[i] if i >= 0 else None for i in oi]
    assert df.Similarity.tolist() == [s if i >= 0 else 0.0 for s, i in zip(os_, oi)]   # no /100
    df = RapidFuzz(scorer=name, score_cutoff=0.3, top_n=3).match(FROM, TO, re_train=False)
    assert calls[-1] == ("topk", metric, 0.3, 3, True)
    ti, ts, _ = seq_oracle.topk(metric, FROM, TO, 3, 0.3)
    for r, (tc, sc) in enumerate((("To", "Similarity"), ("To_2", "Similarity_2"), ("To_3", "Similarity_3"))):
        assert df[tc].tolist() == [TO[j] if j >= 0 else None for j in ti[:, r]]
        assert df[sc].tolist() == [v if j >= 0 else 0.0 for v, j in zip(ts[:, r], ti[:, r])]


@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("name", ["indel", "lcsseq", "hamming", "prefix", "postfix"])
def test_editdistance_frames(calls, name, normalize):
    from polyfuzz_b200 import EditDistance
    metric = EditDistance(scorer=name)._metric
    df = EditDistance(scorer=name, normalize=normalize).match(FROM, TO)
    assert calls == [("argbest", metric, float("-inf"), 1, False)]
    oi, os_, _ = seq_oracle.argbest(metric, FROM, TO, float("-inf"))
    assert df.To.tolist() == [TO[i] for i in oi]
    exp = os_ if not normalize else (os_ - os_.min()) / (os_.max() - os_.min())
    np.testing.assert_array_equal(df.Similarity.to_numpy(), exp)
    df = EditDistance(scorer=name, normalize=False).match(FROM)                 # self-match excludes index i only
    oi, os_, _ = seq_oracle.argbest(metric, FROM, FROM, float("-inf"), exclude_self=True)
    assert calls[-1][:3] == ("argbest", metric, float("-inf"))
    assert df.To.tolist() == [FROM[i] for i in oi] and df.Similarity.tolist() == os_.tolist()
    df = EditDistance(scorer=name, normalize=False, top_n=2).match(FROM, TO)
    assert calls[-1] == ("topk", metric, float("-inf"), 2, False)
    ti, _, _ = seq_oracle.topk(metric, FROM, TO, 2, float("-inf"))
    assert df.To_2.tolist() == [TO[j] for j in ti[:, 1]]


def test_candidate_mode_passes_the_metric(monkeypatch):
    from polyfuzz_b200 import editdist
    from polyfuzz_b200.matchers import _rapidfuzz
    seen = []

    class Candidates:
        def match_arrays(self, from_list, to_list, re_train):
            return torch.tensor([[1, -1], [0, 2]], dtype=torch.int32), None, None

    def edit_cand_topk(frm, to, cand, k, metric="ratio", score_cutoff=0.0, exclude_self=False, kept=None, reuse=False):
        seen.append((cand.tolist(), k, metric, score_cutoff, exclude_self, reuse))
        return torch.tensor([[1, -1], [2, 0]], dtype=torch.int32), torch.tensor([[0.5, 0.0], [0.75, 0.25]])

    monkeypatch.setattr(editdist, "edit_cand_topk", edit_cand_topk)
    idx, score = _rapidfuzz._cand_topk(["ab", "cd"], ["x", "ab", "cd"], "norm_postfix", 0.25, False, 2, Candidates(),
                                       ["x", "ab", "cd"], False, None)
    assert seen == [([[1, -1], [0, 2]], 2, "norm_postfix", 0.25, False, True)]
    assert idx.tolist() == [[1, -1], [2, 0]] and score.tolist() == [[0.5, 0.0], [0.75, 0.25]]


def test_pickle_round_trip():
    from polyfuzz_b200 import EditDistance, RapidFuzz
    for cls, name, metric in ((EditDistance, "lcs_seq", "norm_lcsseq"), (RapidFuzz, "hamming", "norm_hamming"),
                              (EditDistance, "postfix_normalized_similarity", "norm_postfix")):
        m = pickle.loads(pickle.dumps(cls(scorer=name, top_n=3)))
        assert m._metric == metric and m.scorer == name and m.top_n == 3
