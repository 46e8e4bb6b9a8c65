"""Weighted Levenshtein, CPU only: the C oracle (tests/wlev_oracle.c) against a literal transcription of rapidfuzz's pure-Python
Levenshtein with weights, the bounds the kernel derives from the unit distance (DESIGN.md 4.17), the two exact fast paths, the
scorer resolution of functools.partial, the argument rules of pfz_wlev_rows, and the matchers' host logic with the kernels
stubbed."""
import ctypes
import functools
import itertools
import pickle

import numpy as np
import pytest
import torch

import wlev_oracle

GRID = [(0, 0, 0), (0, 1, 1), (1, 0, 3), (1, 1, 0), (1, 3, 2), (5, 2, 7), (1, 1, 2), (3, 3, 9), (2, 2, 2), (65535, 1, 65535)]
ALPHABETS = ["ab", "aé中", "abcdefgh", "abcdefghijkl中"]          # 2, 3, 8 and 13 symbols, some outside ASCII


def uniform_generic(s1, s2, weights):
    """rapidfuzz's _uniform_generic (Levenshtein_py), transcribed; the first row is written i * delete, which the original's
    range(0, (len1 + 1) * delete, delete) equals for delete >= 1 and cannot express for delete = 0."""
    len1 = len(s1)
    insert, delete, replace = weights
    cache = [i * delete for i in range(len1 + 1)]
    for ch2 in s2:
        temp = cache[0]
        cache[0] += insert
        for i in range(len1):
            x = temp
            if s1[i] != ch2:
                x = min(cache[i] + delete, cache[i + 1] + insert, temp + replace)
            temp = cache[i + 1]
            cache[i + 1] = x
    return cache[-1]


def levenshtein_maximum(s1, s2, weights):
    """rapidfuzz's _levenshtein_maximum, transcribed."""
    len1, len2 = len(s1), len(s2)
    insert, delete, replace = weights
    max_dist = len1 * delete + len2 * insert
    if len1 >= len2:
        max_dist = min(max_dist, len2 * replace + (len1 - len2) * delete)
    else:
        max_dist = min(max_dist, len1 * replace + (len2 - len1) * insert)
    return max_dist


def _rand_strings(rng, n, lo, hi, alpha):
    return ["".join(alpha[i] for i in rng.integers(0, len(alpha), rng.integers(lo, hi + 1))) for _ in range(n)]


@pytest.mark.parametrize("weights", GRID)
def test_oracle_equals_transcription(weights):
    rng = np.random.default_rng(sum(weights) % 1000 + 1)
    for alpha in ALPHABETS:
        frm = _rand_strings(rng, 25, 0, 14, alpha) + [""]
        to = _rand_strings(rng, 20, 0, 14, alpha) + [""]
        d, mx = wlev_oracle.wlev_matrix(frm, to, weights)
        for i, a in enumerate(frm):
            for j, b in enumerate(to):
                assert d[i, j] == uniform_generic(a, b, weights), (a, b, weights)
                assert mx[i, j] == levenshtein_maximum(a, b, weights), (a, b, weights)


def test_known_values():
    w = wlev_oracle.wlev
    assert w("kitten", "sitting", (1, 1, 1)) == (3, 7)
    assert w("kitten", "sitting", (1, 1, 2)) == (5, 13)
    assert w("kitten", "sitting", (1, 1, 0)) == (1, 1)
    assert w("kitten", "sitting", (0, 0, 0)) == (0, 0)
    # one insertion is forced; two substitutions beat any deletion, which needs a matching insertion
    assert w("kitten", "sitting", (65535, 1, 65535)) == (3 * 65535, 6 * 65535 + 65535)
    assert w("", "", (5, 2, 7)) == (0, 0) and wlev_oracle.norm_wlev("", "", (5, 2, 7)) == 1.0
    assert w("a", "", (1, 3, 2)) == (3, 3) and w("", "ab", (1, 3, 2)) == (2, 2)
    assert w("a", "b", (1, 3, 2)) == (2, 2) and w("a", "b", (5, 2, 7)) == (7, 7) and w("a", "a", (5, 2, 7)) == (0, 7)
    assert w("ab", "ba", (1, 0, 3)) == (1, 2)                 # a free deletion and one insertion; M = 2 insertions
    assert wlev_oracle.norm_wlev("kitten", "sitting", (1, 1, 2)) == 1.0 - 5 / 13
    assert wlev_oracle.norm_wlev("ab", "ab", (0, 0, 0)) == 1.0


def bounds(L, m, n, weights):
    """The kernel's LB <= D <= UB from the unit distance L (wlev_bounds in csrc/pfz_lev.cu), int64 arrays."""
    wi, wd, ws = (np.int64(x) for x in weights)
    m = m.astype(np.int64); n = n.astype(np.int64)
    dlen = np.abs(m - n); R = L - dlen
    len_cost = dlen * np.where(m >= n, wd, wi)
    pair = wi + wd; s = min(ws, pair)
    M = np.minimum(m * wd + n * wi, np.where(m >= n, n * ws + (m - n) * wd, m * ws + (n - m) * wi))
    lb = len_cost + (R * ws if 2 * ws <= pair else (R * pair + 1) // 2)
    ub = np.minimum(M, len_cost + np.maximum(R * s, R // 2 * pair + (R % 2) * s))
    return lb, ub


BOUND_WEIGHTS = GRID + [(1, 1, 1), (2, 1, 3), (1, 2, 1), (4, 1, 1), (1, 4, 1), (3, 1, 1), (7, 7, 13)]


@pytest.mark.parametrize("weights", BOUND_WEIGHTS)
def test_bounds_chain(weights):
    """LB <= D <= UB on 6 000+ pairs per weight triple, and LB == UB == w * lev for uniform weights."""
    rng = np.random.default_rng(17 + sum(weights) % 977)
    n_pairs = 0
    for alpha in ALPHABETS:
        frm = _rand_strings(rng, 40, 0, 20, alpha) + ["", "a"]
        to = _rand_strings(rng, 40, 0, 20, alpha) + [""]
        D, M = wlev_oracle.wlev_matrix(frm, to, weights)
        L, _ = wlev_oracle.wlev_matrix(frm, to, (1, 1, 1))
        m = np.array([len(s) for s in frm])[:, None] + np.zeros((1, len(to)), np.int64)
        n = np.array([len(s) for s in to])[None, :] + np.zeros((len(frm), 1), np.int64)
        lb, ub = bounds(L, m, n, weights)
        assert (lb <= D).all() and (D <= ub).all() and (ub <= M).all(), weights
        if weights[0] == weights[1] == weights[2]:
            assert (lb == ub).all() and (D == weights[0] * L).all()
        n_pairs += D.size
    assert n_pairs >= 6000


@pytest.mark.parametrize("w", [1, 2, 7, 65535])
def test_uniform_weights_score_as_norm_lev(w):
    """(w, w, w): 1 - (w lev) / (w max) == 1 - lev / max as doubles, so the norm_lev path serves it."""
    rng = np.random.default_rng(w)
    frm = _rand_strings(rng, 60, 0, 30, "abcdé") + [""]
    to = _rand_strings(rng, 60, 0, 30, "abcdé") + [""]
    lev, _ = wlev_oracle.wlev_matrix(frm, to, (1, 1, 1))
    mx = np.maximum(np.array([len(s) for s in frm])[:, None], np.array([len(s) for s in to])[None, :])
    with np.errstate(invalid="ignore", divide="ignore"):
        norm_lev = np.where(mx > 0, 1.0 - lev / mx, 1.0)
    np.testing.assert_array_equal(wlev_oracle.score_matrix(frm, to, (w, w, w)), norm_lev)


def _lcs(a, b):
    prev = [0] * (len(b) + 1)
    for ca in a:
        cur = [0]
        for j, cb in enumerate(b):
            cur.append(prev[j] + 1 if ca == cb else max(prev[j + 1], cur[j]))
        prev = cur
    return prev[-1]


@pytest.mark.parametrize("weights", [(1, 1, 2), (3, 3, 9), (2, 2, 5), (1, 1, 3), (32767, 32767, 65535)])
def test_indel_form_scores_as_indel(weights):
    """(w, w, s >= 2w): D = w * indel and M = w * (m + n), so the score is 1 - indel / (m + n) as a double."""
    _, _, s = weights
    rng = np.random.default_rng(s)
    frm = _rand_strings(rng, 30, 0, 25, "abcé中") + [""]
    to = _rand_strings(rng, 30, 0, 25, "abcé中") + [""]
    got = wlev_oracle.score_matrix(frm, to, weights)
    for i, a in enumerate(frm):
        for j, b in enumerate(to):
            indel = len(a) + len(b) - 2 * _lcs(a, b)
            exp = 1.0 - indel / (len(a) + len(b)) if a or b else 1.0
            assert got[i, j] == exp, (a, b, weights)


def test_oracle_topk_key():
    frm = ["abc", "", "zzz"]
    to = ["abd", "abc", "xbc", "abc", "", "q"]
    for weights in ((1, 1, 1), (5, 2, 7), (1, 0, 3)):
        S = wlev_oracle.score_matrix(frm, to, weights)
        i, s, _ = wlev_oracle.wlev_topk(frm, to, weights, 4, score_cutoff=0.0)
        for r in range(len(frm)):
            c = np.array([j for j in range(len(to)) if S[r, j] >= 0.0])
            c = c[np.lexsort((c, -S[r, c]))][:4]
            assert i[r, :len(c)].tolist() == c.tolist() and s[r, :len(c)].tolist() == S[r, c].tolist()
            assert (i[r, len(c):] == -1).all()
    i, _, _ = wlev_oracle.wlev_topk(to, to, (1, 1, 1), 2, exclude_self=True)
    assert i[1].tolist() == [3, 0] and i[3].tolist() == [1, 0]


# ---- weights and scorer resolution ------------------------------------------------------------------------------------------
def test_check_weights():
    from polyfuzz_b200.editdist import check_weights, uniform_weight
    assert check_weights(None) is None
    assert check_weights((1, 1, 2)) == (1, 1, 2) and check_weights([0, 65535, 3]) == (0, 65535, 3)
    assert check_weights((np.int64(2), np.uint16(3), np.int32(4))) == (2, 3, 4)
    assert all(type(x) is int for x in check_weights((np.int64(2), np.uint16(3), np.int32(4))))
    for bad in ((1, 1), (1, 1, 1, 1), (True, 1, 1), (1, 1, -1), (1, 65536, 1), (1.0, 1, 1), (1, 1, "2"), "abc", 3, {1, 2, 3},
                np.array([1, 1, 1])):
        with pytest.raises(ValueError, match="weights"):
            check_weights(bad)
    assert uniform_weight(None) == 1 and uniform_weight((3, 3, 3)) == 3
    assert uniform_weight((0, 0, 0)) == 0 and uniform_weight((1, 1, 2)) == 0 and uniform_weight((2, 2, 1)) == 0


def _stand_in(name, module):                        # stand-ins with rapidfuzz's function names and module paths
    f = lambda a, b, **kw: 0.0                      # noqa: E731
    f.__name__, f.__module__ = name, module
    return f


def normalized_similarity(s1, s2, weights=None):    # picklable stand-in for rapidfuzz.distance.Levenshtein's
    return 0.0


def test_partial_resolution():
    from polyfuzz_b200 import EditDistance, RapidFuzz
    from polyfuzz_b200.matchers._rapidfuzz import _resolve_scorer
    lev = _stand_in("normalized_similarity", "rapidfuzz.distance.Levenshtein")
    for func in (lev, normalized_similarity, _stand_in("levenshtein", "x"), _stand_in("normalized_levenshtein", "x"),
                 _stand_in("normalized_similarity", "rapidfuzz.distance.DamerauLevenshtein")):
        for weights, metric in (((1, 1, 2), "wlev"), ((5, 2, 7), "wlev"), ((0, 0, 0), "wlev"), ((3, 3, 3), "norm_lev"),
                                (None, "norm_lev")):
            p = functools.partial(func, weights=weights)
            assert _resolve_scorer(p, "ratio") == metric and _resolve_scorer(p, "WRatio", allow_jaro=True) == metric
            for cls in (EditDistance, RapidFuzz):
                m = cls(scorer=p)
                assert m._metric == metric and m._weights == (None if weights is None else tuple(weights))
        assert _resolve_scorer(functools.partial(func), "ratio") == "norm_lev"
    # positional arguments, other keywords, and partials of any other scorer
    refused = [functools.partial(lev, "a"), functools.partial(lev, weights=(1, 1, 2), processor=str.lower),
               functools.partial(lev, score_cutoff=0.5), functools.partial(_stand_in("ratio", "rapidfuzz.fuzz"), weights=(1, 1, 2)),
               functools.partial(_stand_in("WRatio", "rapidfuzz.fuzz"), weights=(1, 1, 2)),
               functools.partial(_stand_in("normalized_similarity", "rapidfuzz.distance.OSA"), weights=(1, 1, 2)),
               functools.partial(_stand_in("jaro_winkler_similarity", "jellyfish"), weights=(1, 1, 2)),
               functools.partial(_stand_in("dl", "x"), weights=(1, 1, 2)), functools.partial(_stand_in("mystery", "x")),
               functools.partial(lambda a, b: 0.0, weights=(1, 1, 2))]
    for p in refused:
        for cls in (EditDistance, RapidFuzz):
            with pytest.raises(NotImplementedError, match="partial"):
                cls(scorer=p)
        with pytest.raises(NotImplementedError):
            _resolve_scorer(p, "ratio", allow_jaro=True)
    for bad in ((1, 1), (1, 1, 65536), (True, 1, 1), (1.5, 1, 1), (-1, 1, 1)):
        for cls in (EditDistance, RapidFuzz):
            with pytest.raises(ValueError, match="weights"):
                cls(scorer=functools.partial(lev, weights=bad))


def test_existing_names_keep_their_metric():
    from polyfuzz_b200 import fuzzy
    from polyfuzz_b200.matchers._rapidfuzz import _JARO, _NAMES, _resolve_scorer
    for name, metric in _NAMES.items():
        assert _resolve_scorer(name, "ratio") == metric
        assert _resolve_scorer(_stand_in(name, "somewhere"), "ratio") == metric
    for name, metric in _JARO.items():
        assert _resolve_scorer(name, "ratio", allow_jaro=True) == metric
    for name in fuzzy.SCORER:
        assert _resolve_scorer(name, "ratio") == name
    assert _resolve_scorer(_stand_in("normalized_similarity", "rapidfuzz.distance.OSA"), "ratio") == "norm_osa"
    assert _resolve_scorer(None, "ratio") == "ratio" and _resolve_scorer(None, "WRatio") == "WRatio"


def test_metric_tuples_unchanged():
    from polyfuzz_b200 import editdist
    assert "wlev" not in editdist.METRIC and "wlev" not in editdist.TOPK_METRICS
    with pytest.raises(ValueError, match="matrix"):
        editdist.edit_wlev_argbest_staged(None, None, (1, 1, 2), want_matrix=True)


def test_pickle_round_trip():
    from polyfuzz_b200 import EditDistance, RapidFuzz
    for cls in (EditDistance, RapidFuzz):
        m = cls(scorer=functools.partial(normalized_similarity, weights=(5, 2, 7)))
        m2 = pickle.loads(pickle.dumps(m))
        assert m2._metric == "wlev" and m2._weights == (5, 2, 7)
        assert m2.scorer.func is normalized_similarity and m2.scorer.keywords == {"weights": (5, 2, 7)}


# ---- pfz_wlev_rows argument rules (n_ids = 0, null buffers: nothing is read) -------------------------------------------------
BUF = np.zeros(64, dtype=np.int64)
NN = ctypes.c_void_p(BUF.ctypes.data)
SOURCES = [(None, 1, 0, None), (None, 3, 0, None), (None, 0, 0, None), (NN, 1, 4, NN), (NN, 2, 4, NN), (NN, 1, 0, NN),
           (NN, 1, 4, None)]


def test_wlev_rows_rules():
    from polyfuzz_b200 import _lib
    lib = _lib.load()
    n_allowed = 0
    for weights, n_words, k, part_dist, source in itertools.product(
            ((1, 1, 2), (0, 0, 0), (65535, 65535, 65535), (-1, 1, 1), (1, 65536, 1), (1, 1, -3)), (-1, 0, 1, 3, 16, 32),
            (-1, 0, 1, 32, 33), (False, True), SOURCES):
        cand, n_splits, c, pos_of = source
        rc = lib.pfz_wlev_rows(NN, NN, 10, NN, 0, n_words, NN, NN, NN, NN, NN, 20, *weights, 0.5, 0, 0, n_splits, k, cand, c, pos_of,
                               NN, NN, NN if part_dist else None, NN, None)
        broken = []
        if cand is not None:
            broken += ["candidate mode"] if n_splits != 1 or c < 1 or pos_of is None else []
        elif n_splits < 1:
            broken.append("n_splits < 1")
        if not all(0 <= w <= 65535 for w in weights):
            broken.append("weights")
        if n_words not in (0, 1, 2, 4, 8, 16):
            broken.append("n_words")
        if not 0 <= k <= 32:
            broken.append(f"k={k} unsupported")
        elif k >= 1 and part_dist:
            broken.append("top-k has no distance output")
        elif k == 0 and not part_dist:
            broken.append("arg-best needs part_dist")
        msg = lib.pfz_last_error().decode()
        if not broken:
            assert rc == 0, (weights, n_words, k, part_dist, source, msg)
            n_allowed += 1
        else:
            assert rc == 1 and any(b in msg for b in broken), (weights, n_words, k, part_dist, source, broken, msg)
    assert n_allowed > 50


# ---- matcher host logic with the kernels stubbed ------------------------------------------------------------------------------
@pytest.fixture
def calls(monkeypatch):
    from polyfuzz_b200 import editdist
    seen = []

    def edit_wlev_argbest(frm, to, weights, score_cutoff=0.0, exclude_self=False, **kw):
        seen.append(("argbest", weights, float(score_cutoff), 1, kw.get("reuse")))
        i, s, d = wlev_oracle.wlev_argbest(frm, to, weights, score_cutoff, exclude_self)
        return torch.from_numpy(i.copy()), torch.from_numpy(s.copy()), torch.from_numpy(d.astype(np.int32))

    def edit_wlev_topk(frm, to, k, weights, score_cutoff=0.0, exclude_self=False, **kw):
        seen.append(("topk", weights, float(score_cutoff), k, kw.get("reuse")))
        i, s, _ = wlev_oracle.wlev_topk(frm, to, weights, k, score_cutoff, exclude_self)
        return torch.from_numpy(i), torch.from_numpy(s)

    def edit_argbest(frm, to, metric="ratio", score_cutoff=0.0, exclude_self=False, **kw):
        seen.append(("norm_lev argbest", metric, float(score_cutoff), 1, kw.get("reuse")))
        i, s, d = wlev_oracle.wlev_argbest(frm, to, None, score_cutoff, exclude_self)
        return torch.from_numpy(i.copy()), torch.from_numpy(s.copy()), torch.from_numpy(d.astype(np.int32))

    monkeypatch.setattr(editdist, "edit_wlev_argbest", edit_wlev_argbest)
    monkeypatch.setattr(editdist, "edit_wlev_topk", edit_wlev_topk)
    monkeypatch.setattr(editdist, "edit_argbest", edit_argbest)
    return seen


FROM = ["kitten", "Jhon Smtih", "Micorsoft", "apple", "appel", "house", ""]
TO = ["sitting", "XY", "Joan Smyth", "John Smith", "Microsoft", "apple", "apples", "mouse"]


def test_rapidfuzz_frames(calls):
    from polyfuzz_b200 import RapidFuzz
    p = functools.partial(normalized_similarity, weights=(5, 2, 7))
    df = RapidFuzz(scorer=p, score_cutoff=0.6).match(FROM, TO)
    assert calls == [("argbest", (5, 2, 7), 0.6, 1, False)]              # the cutoff on 0..1, as norm_lev
    oi, os_, _ = wlev_oracle.wlev_argbest(FROM, TO, (5, 2, 7), 0.6)
    assert df.To.tolist() == [TO[i] if i >= 0 else None for i in oi]
    assert df.Similarity.tolist() == [s if i >= 0 else 0.0 for s, i in zip(os_, oi)]   # no /100
    df = RapidFuzz(scorer=p, score_cutoff=0.5, top_n=3).match(FROM, TO, re_train=False)
    assert calls[-1] == ("topk", (5, 2, 7), 0.5, 3, True)
    ti, ts, _ = wlev_oracle.wlev_topk(FROM, TO, (5, 2, 7), 3, 0.5)
    for r, (tc, sc) in enumerate((("To", "Similarity"), ("To_2", "Similarity_2"), ("To_3", "Similarity_3"))):
        assert df[tc].tolist() == [TO[j] if j >= 0 else None for j in ti[:, r]]
        assert df[sc].tolist() == [v if j >= 0 else 0.0 for v, j in zip(ts[:, r], ti[:, r])]
    RapidFuzz(scorer=functools.partial(normalized_similarity, weights=(2, 2, 2)), score_cutoff=0.6).match(FROM, TO)
    assert calls[-1] == ("norm_lev argbest", "norm_lev", 0.6, 1, False)


@pytest.mark.parametrize("normalize", [False, True])
def test_editdistance_frames(calls, normalize):
    from polyfuzz_b200 import EditDistance
    p = functools.partial(normalized_similarity, weights=(1, 3, 2))
    df = EditDistance(scorer=p, normalize=normalize).match(FROM, TO)
    assert calls == [("argbest", (1, 3, 2), float("-inf"), 1, False)]
    oi, os_, _ = wlev_oracle.wlev_argbest(FROM, TO, (1, 3, 2), float("-inf"))
    exp = os_ if not normalize else (os_ - os_.min()) / (os_.max() - os_.min())
    assert df.To.tolist() == [TO[i] for i in oi]
    np.testing.assert_array_equal(df.Similarity.to_numpy(), exp)
    df = EditDistance(scorer=p, normalize=False).match(FROM)                   # self-match excludes index i only
    oi, os_, _ = wlev_oracle.wlev_argbest(FROM, FROM, (1, 3, 2), float("-inf"), exclude_self=True)
    assert calls[-1][:3] == ("argbest", (1, 3, 2), float("-inf"))
    assert df.To.tolist() == [FROM[i] for i in oi] and df.Similarity.tolist() == os_.tolist()
    df = EditDistance(scorer=p, normalize=False, top_n=2).match(FROM, TO)
    assert calls[-1] == ("topk", (1, 3, 2), float("-inf"), 2, False)
    ti, _, _ = wlev_oracle.wlev_topk(FROM, TO, (1, 3, 2), 2, float("-inf"))
    assert df.To_2.tolist() == [TO[j] for j in ti[:, 1]]


def test_candidate_mode_passes_the_weights(monkeypatch):
    from polyfuzz_b200 import editdist
    from polyfuzz_b200.matchers import _rapidfuzz
    seen = []

    class Candidates:
        def match_arrays(self, from_list, to_list, re_train):
            return torch.tensor([[1, -1], [0, 2]], dtype=torch.int32), None, None

    def edit_wlev_cand_topk(frm, to, cand, k, weights, score_cutoff=0.0, exclude_self=False, kept=None, reuse=False):
        seen.append((cand.tolist(), k, weights, score_cutoff, exclude_self, reuse))
        return torch.tensor([[1, -1], [2, 0]], dtype=torch.int32), torch.tensor([[0.5, 0.0], [0.75, 0.25]])

    monkeypatch.setattr(editdist, "edit_wlev_cand_topk", edit_wlev_cand_topk)
    idx, score = _rapidfuzz._cand_topk(["ab", "cd"], ["x", "ab", "cd"], "wlev", 0.25, False, 2, Candidates(), ["x", "ab", "cd"],
                                       False, None, weights=(5, 2, 7))
    assert seen == [([[1, -1], [0, 2]], 2, (5, 2, 7), 0.25, False, True)]
    assert idx.tolist() == [[1, -1], [2, 0]] and score.tolist() == [[0.5, 0.0], [0.75, 0.25]]
