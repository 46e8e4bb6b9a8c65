"""GPU tests of every edit-distance scorer at score cutoffs equal to achieved scores and one ulp either side of them.

rapidfuzz applies the cutoff c of fuzz.ratio and partial_ratio in two steps (ns >= c/100, then ns*100 >= c; see
tests/cutoff_cases.py), and a pair whose score s has (s/100) > ns is rejected at c = s although it scores s at c = 0.  K3
(ratio) and K3b (the partial steps of partial_ratio, partial_token_*, WRatio) must reject it too.  The 0..1 metrics
(norm_lev, norm_osa, norm_dl, jaro, jaro_winkler) test score >= c once: a pair at c = s is kept.

Expected values come from the oracle's score matrix evaluated at the same cutoff, sorted by (score desc, index asc) over the
candidates score >= cutoff; arg-best results are also checked against oracle.fuzz.extract_one.  Indices and scores are compared
with ==.  oracle.fuzz.lcs_len is swapped for the C LCS of tests/lcs_oracle.c (memoised) in this module only."""
import collections
import functools
import math
import multiprocessing
import os
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

import cutoff_cases as cc
import dl_oracle
import jaro_oracle
import lcs_oracle
import osa_oracle
from oracle import fuzz as ofuzz
from oracle import native as onative

pytestmark = pytest.mark.gpu
NT = os.cpu_count() or 1
KS = (1, 5, 32)
SPLITS = (1, 3, None)
WORDS = ["The", "of", "and", "a", "Night", "Day", "Love", "Man", "Last", "Story", "Dead", "II", "Return", "King", "night", "é",
         "Noël", "x", "ab", "ba", "abc", "cab", "c", "b"]


@pytest.fixture(scope="module", autouse=True)
def c_lcs():
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ofuzz, "lcs_len", functools.lru_cache(maxsize=None)(lcs_oracle.lcs_len))
        yield


@pytest.fixture(scope="module")
def ed():
    from polyfuzz_b200 import editdist
    return editdist


@pytest.fixture(scope="module")
def fz():
    from polyfuzz_b200 import fuzzy
    return fuzzy


def score_matrix(frm, to, scorer, cutoff):
    fn = ofuzz.SCORERS[scorer]
    return np.array([[fn(a, b, cutoff) for b in to] for a in frm], dtype=np.float64).reshape(len(frm), len(to))


def oracle_topk(S, k, cutoff):
    """Rows of S sorted by (score desc, index asc) over the candidates score >= cutoff."""
    n, m = S.shape
    oi = np.full((n, k), -1, np.int32); ov = np.zeros((n, k))
    cols = np.arange(m)
    for i in range(n):
        c = cols[S[i] >= cutoff]
        order = np.lexsort((c, -S[i, c]))[:k]
        oi[i, :len(order)] = c[order]; ov[i, :len(order)] = S[i, c[order]]
    return oi, ov


def _eq(got, exp, what):
    np.testing.assert_array_equal(got[0].cpu().numpy(), exp[0], err_msg=f"indices, {what}")
    np.testing.assert_array_equal(got[1].cpu().numpy(), exp[1], err_msg=f"scores, {what}")


def check(argbest, topk, S, cutoff, extract=None):
    """argbest(n_splits) -> (idx, score, ...), topk(k, n_splits) -> (idx, score) at every split count and k against S (the
    oracle's matrix at this cutoff); extract: the oracle's extractOne per row, (index, score) or None."""
    ei, ev = oracle_topk(S, 1, cutoff)
    for n_splits in SPLITS:
        bi, bs = argbest(n_splits)[:2]
        _eq((bi, bs), (ei[:, 0], ev[:, 0]), f"arg-best, cutoff {cutoff!r}, n_splits {n_splits}")
        for k in KS:
            _eq(topk(k, n_splits), oracle_topk(S, k, cutoff), f"top-{k}, cutoff {cutoff!r}, n_splits {n_splits}")
    if extract is not None:
        got = [(int(i), float(s)) if i >= 0 else None for i, s in zip(bi.cpu().numpy(), bs.cpu().numpy())]
        assert got == extract, f"arg-best against extractOne, cutoff {cutoff!r}"


def titles(rng, n, lo=1, hi=6):
    return [" ".join(rng.choice(WORDS, rng.integers(lo, hi + 1))) for _ in range(n)]


# ---- K3, ratio: lists built from boundary (|a|, |b|, lcs) triples ------------------------------------------------------------------
def _ratio_families():
    """(m, d) with ns = 1 - d/m a boundary value: 17/25 (68.0) at m = 50 and m = 150 (from-strings past 64 code points), and
    the first two other boundary values at m = 40..60."""
    fams = [(50, 16), (150, 48)]
    seen = {cc.ratio_ns(25, 25, 17)}
    for m in range(40, 61):
        for d in range(m % 2, m + 1, 2):
            ns = cc.ratio_ns(m - m // 2, m // 2, (m - d) // 2)
            if len(fams) < 4 and 0.3 < ns < 0.95 and ns not in seen and cc.is_boundary_score(ns):
                fams.append((m, d)); seen.add(ns)
    return fams


_RATIO = {}


def ratio_lists():
    """Per family (its own three letters, so families do not match each other): from-strings of 6 lengths; to-strings at the
    exact partner length (twice), one longer and one shorter, and with one more and one fewer shared letter -- each row has
    candidates at the family's value and next to it.  Mixed with random filler, to-list shuffled."""
    if not _RATIO:
        rng = np.random.default_rng(41)
        fams = _ratio_families()
        frm, to = [], []
        for f, (m, d) in enumerate(fams):
            x, y, z = (chr(0x61 + 3 * f + i) for i in range(3))
            lcs = (m - d) // 2
            for la in np.linspace(max(lcs, 1), m - lcs, 6).astype(int):
                lb = m - la
                a, b = cc.ratio_strings(la, lb, lcs, x, y, z)
                frm.append(a)
                to += [b, b, b + z, b[:-1] if lb > lcs else b + z + z, x + b, b[1:] + z]
        filler = ["".join(rng.choice(list("abcdefghijkl"), rng.integers(1, 60))) for _ in range(60)]
        frm += filler[:10]
        to += filler[10:]
        rng.shuffle(to)
        _RATIO.update(frm=frm, to=list(to), fams=fams)
    return _RATIO["frm"], _RATIO["to"], _RATIO["fams"]


@pytest.mark.parametrize("family", range(4))
def test_k3_ratio_at_boundary_scores(ed, family):
    frm, to, fams = ratio_lists()
    m, d = fams[family]
    s = cc.ratio_ns(m - m // 2, m // 2, (m - d) // 2) * 100.0
    S0 = score_matrix(frm, to, "ratio", 0.0)
    n_at = int((S0 == s).sum())
    assert n_at >= 6 and (score_matrix(frm, to, "ratio", s)[S0 == s] == 0).all()     # boundary pairs: rejected at c = s
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    for c in cc.neighbours(s):
        S = score_matrix(frm, to, "ratio", c)
        ext = [None if e is None else (e[2], e[1]) for e in (ofuzz.extract_one(a, to, ofuzz.ratio, c) for a in frm)]
        check(lambda ns: ed.edit_argbest_staged(Q, T, "ratio", c, n_splits=ns),
              lambda k, ns: ed.edit_topk_staged(Q, T, k, "ratio", c, n_splits=ns), S, c, ext)


# ---- K3b, every scorer: boundary pairs and titles, in word class 1 and one CTA per row (257..512 code points) ---------------------
FUZZ_SCORERS = ["ratio", "QRatio", "partial_ratio", "token_sort_ratio", "token_set_ratio", "token_ratio", "partial_token_sort_ratio",
                "partial_token_set_ratio", "partial_token_ratio", "WRatio"]
_FZ = {}


def short_lists(scorer):
    """Word class 1: 8 of the scorer's boundary pairs (token_set_ratio has none: token_sort_ratio's), 8 + 24 titles."""
    if scorer not in _FZ:
        src = "token_sort_ratio" if scorer == "token_set_ratio" else scorer
        pairs = cc.boundary_pairs(src, 8, seed=FUZZ_SCORERS.index(scorer) + 100)
        rng = np.random.default_rng(FUZZ_SCORERS.index(scorer))
        frm = [a for a, _, _ in pairs] + titles(rng, 8)
        to = [b for _, b, _ in pairs] + titles(rng, 24) + [pairs[0][1], pairs[3][1]]
        order = rng.permutation(len(to))
        _FZ[scorer] = (frm, [to[j] for j in order])
    return _FZ[scorer]


def long_lists():
    """One CTA per row: from-strings of 260, 380 and 500 code points over "abc " (partial_ratio skips the windows that end on a
    'c' against to-strings over "ab "), to-strings of 4..40 code points over "ab " and "abc ", and one of 300."""
    if "long" not in _FZ:
        rng = np.random.default_rng(77)
        rnd = lambda alpha, n: "".join(rng.choice(list(alpha), n)).strip() or alpha[0]  # noqa: E731
        frm = [rnd("abc ", n) for n in (262, 384, 505)]
        assert all(257 <= len(s) <= 512 for s in frm)
        to = [rnd("ab " if j % 2 else "abc ", int(rng.integers(4, 41))) for j in range(40)] + [rnd("abc ", 300)]
        _FZ["long"] = (frm, to)
    return _FZ["long"]


def boundary_cutoffs(frm, to, scorer, S0, n=3):
    """The n most frequent scores of S0 at which some pair is rejected (boundary), or, when there are none, the n most frequent
    positive scores; each with its neighbours.  Also returns whether boundary scores were found."""
    fn = ofuzz.SCORERS[scorer]
    bnd = collections.Counter(S0[i, j] for i in range(S0.shape[0]) for j in range(S0.shape[1])
                              if 0 < S0[i, j] < 100 and fn(frm[i], to[j], S0[i, j]) == 0)
    found = bool(bnd)
    if not bnd:
        bnd = collections.Counter(v for v in S0.ravel() if 0 < v < 100)
    vals = sorted(v for v, _ in bnd.most_common(n))
    return [c for v in vals for c in cc.neighbours(v)], found


@pytest.mark.parametrize("cls", ["word_class_1", "cta_row"])
@pytest.mark.parametrize("scorer", FUZZ_SCORERS)
def test_k3b_at_boundary_scores(fz, scorer, cls):
    frm, to = short_lists(scorer) if cls == "word_class_1" else long_lists()
    fn = ofuzz.SCORERS[scorer]
    S0 = score_matrix(frm, to, scorer, 0.0)
    cutoffs, found = boundary_cutoffs(frm, to, scorer, S0)
    if cls == "word_class_1":
        assert found == (scorer != "token_set_ratio")
    elif scorer in ("partial_ratio", "partial_token_sort_ratio"):
        assert found, "the long lists hold no boundary pair"
    for c in cutoffs:
        S = score_matrix(frm, to, scorer, c)
        ext = [None if e is None else (e[2], e[1]) for e in (ofuzz.extract_one(a, to, fn, c) for a in frm)]
        check(lambda ns: fz.fuzz_argbest(frm, to, scorer, c, n_splits=ns),
              lambda k, ns: fz.fuzz_topk(frm, to, k, scorer, c, n_splits=ns), S, c, ext)


# ---- K3, the 0..1 metrics: one test, score >= cutoff ------------------------------------------------------------------------------
_UNIT = {}


def unit_lists():
    if not _UNIT:
        rng = np.random.default_rng(5)
        rnd = lambda n, lo, hi: ["".join(rng.choice(list("abc"), rng.integers(lo, hi + 1))) for _ in range(n)]  # noqa: E731
        frm = rnd(40, 2, 9) + ["ca", "abc", ""]
        to = rnd(200, 1, 10) + ["abc", "ac", "", "ca"]
        _UNIT.update(frm=frm, to=to)
    return _UNIT["frm"], _UNIT["to"]


def unit_matrix(frm, to, metric):
    if metric in ("jaro", "jaro_winkler"):
        w = metric == "jaro_winkler"
        return np.array([[jaro_oracle.jaro_pair(a, b, winkler=w)[0] for b in to] for a in frm], dtype=np.float64)
    if metric == "norm_lev":
        d = onative.editdist_matrix(frm, to, "lev", n_threads=NT)
    elif metric == "norm_osa":
        d = osa_oracle.osa_matrix(frm, to, n_threads=NT)
    else:
        d = dl_oracle.dl_matrix(frm, to, n_threads=NT)
    la = np.array([len(s) for s in frm], dtype=np.float64)[:, None]
    lb = np.array([len(s) for s in to], dtype=np.float64)[None, :]
    m = np.maximum(la, lb)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(m > 0, 1.0 - d.astype(np.float64) / m, 1.0)


@pytest.mark.parametrize("metric", ["norm_lev", "norm_osa", "norm_dl", "jaro", "jaro_winkler"])
def test_unit_metrics_keep_the_cutoff_score(ed, metric):
    frm, to = unit_lists()
    S = unit_matrix(frm, to, metric)
    fifth = oracle_topk(S, 5, 0.0)[1][:, 4:5]                      # each row's 5th best score
    vals = collections.Counter(S[(S >= fifth) & (S > 0) & (S < 1)])
    picks = [v for v, _ in vals.most_common(2)]
    if metric == "norm_dl":
        # DL scores that only DL reaches (a swapped pair edited again): at such a cutoff, a row with fewer than k OSA candidates
        # has its gate at the cutoff, and these pairs tie it (the gate keeps ub == gate)
        SO = unit_matrix(frm, to, "norm_osa")
        dl_only = collections.Counter(S[(S > SO) & (S >= fifth)])
        picks.append(dl_only.most_common(1)[0][0])
        ties = 0
        for c in picks:
            for k in KS:
                for r in range(len(frm)):
                    so = np.sort(SO[r][SO[r] >= c])[::-1]
                    gate = so[k - 1] if len(so) >= k else c
                    ties += int(((S[r] == gate) & (SO[r] < gate)).sum())
        assert ties > 0
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    for v in picks:
        assert (oracle_topk(S, 32, v)[1] == v).any()      # equality keeps: pairs at v are among the expected results at c = v
        for c in cc.neighbours(v):
            check(lambda ns: ed.edit_argbest_staged(Q, T, metric, c, n_splits=ns),
                  lambda k, ns: ed.edit_topk_staged(Q, T, k, metric, c, n_splits=ns), S, c)


# ---- the matchers -----------------------------------------------------------------------------------------------------------------
def _expected_frame(frm, to, S, cutoff, top_n):
    """The reference's frame: per row the extractOne / extract(limit=top_n) result, score / 100; (None, 0.0) where nothing passes."""
    oi, ov = oracle_topk(S, top_n, cutoff)
    cols = {}
    for r in range(top_n):
        cols["To" if r == 0 else f"To_{r + 1}"] = [to[j] if j >= 0 else None for j in oi[:, r]]
        cols["Similarity" if r == 0 else f"Similarity_{r + 1}"] = [v / 100 if j >= 0 else 0.0 for j, v in zip(oi[:, r], ov[:, r])]
    return cols


def _frame_eq(got, exp):
    for name, col in exp.items():
        assert got[name].tolist() == col, name


def test_matchers_at_boundary_cutoffs():
    from polyfuzz_b200 import RapidFuzz
    frm, to, _ = ratio_lists()
    assert 0.68 * 100 == 68.0
    S = score_matrix(frm, to, "ratio", 68.0)
    exp1 = [ofuzz.extract_one(a, to, ofuzz.ratio, 68.0) for a in frm]
    got = RapidFuzz(scorer="ratio", score_cutoff=0.68).match(frm, to)
    assert got.To.tolist() == [None if e is None else e[0] for e in exp1]
    assert got.Similarity.tolist() == [0.0 if e is None else e[1] / 100 for e in exp1]
    _frame_eq(RapidFuzz(scorer="ratio", score_cutoff=0.68, top_n=3).match(frm, to), _expected_frame(frm, to, S, 68.0, 3))

    frm, to = short_lists("partial_ratio")
    S0 = score_matrix(frm, to, "partial_ratio", 0.0)
    rejected = 0
    for s in sorted({s for _, _, s in cc.boundary_pairs("partial_ratio", 8, seed=FUZZ_SCORERS.index("partial_ratio") + 100)}):
        u = s / 100
        c = u * 100                                      # what the matcher hands to the scorer
        S = score_matrix(frm, to, "partial_ratio", c)
        rejected += int(((S0 >= c) & (S == 0)).sum())
        for top_n in (1, 3):
            got = RapidFuzz(scorer="partial_ratio", score_cutoff=u, top_n=top_n).match(frm, to)
            _frame_eq(got, _expected_frame(frm, to, S, c, top_n))
    assert rejected > 0                                  # some pair scores >= c at cutoff 0 and is rejected at c


# ---- WRatio at cutoff 0 on real movie titles --------------------------------------------------------------------------------------
def test_wratio_real_movie_titles(fz):
    """WRatio threads max(c, end_ratio)/0.9 and /0.95 down to its partial steps, so even at cutoff 0 the two-step rule decides
    scores and winners.  Sampled Netflix rows against a slice of the IMDB list, oracle in a process pool."""
    from polyfuzz_b200 import datasets
    data, kind = datasets.load_movie_titles()
    if kind != "real":
        pytest.skip("the movie-title fixture is not present")
    rng = np.random.default_rng(2026)
    rows = np.sort(rng.choice(len(data["Netflix"]), 48, replace=False))
    frm = [data["Netflix"][i] for i in rows]
    to = data["IMDB"][:5000]
    with ProcessPoolExecutor(max_workers=min(NT, 16), mp_context=multiprocessing.get_context("spawn")) as ex:
        S = np.array(list(ex.map(cc.wratio_row, [(a, to) for a in frm])), dtype=np.float64)
    bi, bs = fz.fuzz_argbest(frm, to, "WRatio")
    ei, ev = oracle_topk(S, 1, 0.0)
    _eq((bi, bs), (ei[:, 0], ev[:, 0]), "WRatio arg-best")
    _eq(fz.fuzz_topk(frm, to, 10, "WRatio"), oracle_topk(S, 10, 0.0), "WRatio top-10")
