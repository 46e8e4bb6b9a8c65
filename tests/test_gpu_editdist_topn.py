"""GPU tests of the top-k epilogue of K3 / K3b (pfz_lev_topk, pfz_fuzz_topk) and of RapidFuzz / EditDistance with top_n > 1.
The oracle is a full score matrix sorted by the canonical key (score desc, to-index asc): ratio / norm_lev from the
Wagner-Fischer distances of oracle.native with the kernel's IEEE expressions (numpy has no FMA, so they are exact), the
K3b scorers from oracle/fuzz.py, Jaro from tests/jaro_oracle.py.  Indices and scores are compared with ==."""
import os

import numpy as np
import pandas as pd
import pytest

import jaro_oracle
from oracle import fuzz as ofuzz
from oracle import native as onative

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
REF = os.path.join(ROOT, "oracle", "_ref")
NT = os.cpu_count() or 1
KS = [2, 3, 10, 31, 32]
FROM = ["apple", "apples", "appl", "recal", "house", "similarity"]
TO = ["apple", "apples", "mouse"]


@pytest.fixture(scope="module")
def ed():
    from polyfuzz_b200 import editdist
    return editdist


@pytest.fixture(scope="module")
def fz():
    from polyfuzz_b200 import fuzzy
    return fuzzy


def _rand_strings(rng, n, lo, hi, alpha):
    return ["".join(alpha[i] for i in rng.integers(0, len(alpha), rng.integers(lo, hi + 1))) for _ in range(n)]


def score_matrix(frm, to, metric):
    """float64 [n_from, n_to] of the metric, exactly as the kernels compute it."""
    if metric in ("ratio", "norm_lev"):
        d = onative.editdist_matrix(frm, to, "indel" if metric == "ratio" else "lev", n_threads=NT).astype(np.float64)
        la = np.array([len(s) for s in frm], dtype=np.float64)[:, None]
        lb = np.array([len(s) for s in to], dtype=np.float64)[None, :]
        if metric == "ratio":
            m = la + lb
            with np.errstate(invalid="ignore", divide="ignore"):
                return np.where(m > 0, (1.0 - d / m) * 100.0, 100.0)
        m = np.maximum(la, lb)
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where(m > 0, 1.0 - d / m, 1.0)
    if metric in ("jaro", "jaro_winkler"):
        w = metric == "jaro_winkler"
        return np.array([[jaro_oracle.jaro_pair(a, b, winkler=w)[0] for b in to] for a in frm], dtype=np.float64)
    fn = ofuzz.SCORERS[metric]
    return np.array([[fn(a, b) for b in to] for a in frm], dtype=np.float64)


def oracle_topk(S, k, cutoff=float("-inf"), exclude_self=False):
    """Rows of S sorted by (score desc, index asc) over the candidates score >= cutoff (and j != i in a self-match)."""
    n, m = S.shape
    oi = np.full((n, k), -1, np.int32); ov = np.zeros((n, k))
    cols = np.arange(m)
    for i in range(n):
        ok = S[i] >= cutoff
        if exclude_self and i < m:
            ok[i] = False
        c = cols[ok]
        order = np.lexsort((c, -S[i, c]))[:k]
        oi[i, :len(order)] = c[order]; ov[i, :len(order)] = S[i, c[order]]
    return oi, ov


def _eq(got, exp):
    gi, gv = got
    np.testing.assert_array_equal(gi.cpu().numpy(), exp[0])
    np.testing.assert_array_equal(gv.cpu().numpy(), exp[1])


# ---- K3: every word class, n_splits 1 / 3 / default ------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["ratio", "norm_lev", "jaro", "jaro_winkler"])
@pytest.mark.parametrize("lo,hi,n_from,n_to", [(0, 12, 70, 150), (20, 40, 70, 150), (50, 70, 40, 100), (90, 140, 30, 90),
                                               (200, 300, 20, 60), (500, 600, 10, 40), (900, 1024, 6, 24)])
def test_k3_every_word_class(ed, metric, lo, hi, n_from, n_to):
    rng = np.random.default_rng(lo * 7 + hi)
    alpha = "abcdefgh éß中K"
    frm = _rand_strings(rng, n_from, lo, hi, alpha) + ["", "a"]
    to = _rand_strings(rng, n_to, max(0, lo // 2), hi + 10, alpha) + ["", frm[3], frm[3][:-1] if frm[3] else "x"]
    S = score_matrix(frm, to, metric)
    cut = 0.0 if metric in ("ratio", "norm_lev") else float("-inf")
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    for k in KS:
        exp = oracle_topk(S, k, cut)
        for n_splits in (1, 3, None):
            _eq(ed.edit_topk_staged(Q, T, k, metric, cut, n_splits=n_splits), exp)
    # column 1 is the arg-best
    bi, bs, _ = ed.edit_argbest_staged(Q, T, metric, cut)
    ti, tv = ed.edit_topk_staged(Q, T, 10, metric, cut)
    np.testing.assert_array_equal(ti[:, 0].cpu().numpy(), bi.cpu().numpy())
    np.testing.assert_array_equal(tv[:, 0].cpu().numpy(), bs.cpu().numpy())


def test_k3_alphabet_batches(ed):
    big = [chr(0x4E00 + i) + chr(0x4E00 + (i * 7) % 600) + "ab" for i in range(600)]
    to = big[::3] + ["ab", "中ab"]
    for metric in ("norm_lev", "jaro_winkler"):
        S = score_matrix(big, to, metric)
        for k in (3, 32):
            _eq(ed.edit_topk(big, to, k, metric, 0.0), oracle_topk(S, k, 0.0))


# ---- K3b: every scorer ---------------------------------------------------------------------------------------------------
WORDS = ["The", "of", "and", "a", "Night", "Day", "Love", "Man", "Last", "Story", "Dead", "II", "Return", "King", "night", "é", "Noël",
         "x", "Zorro", "Christmas", "Carol", "day", "man", "House", "Home"]


def _titles(rng, n, lo=1, hi=6):
    out = []
    for _ in range(n):
        ws = list(rng.choice(WORDS, rng.integers(lo, hi + 1)))
        if rng.random() < 0.15:
            ws.append(ws[0])
        s = " ".join(ws)
        if rng.random() < 0.1:
            s = s.replace(" ", "  ", 1) + " "
        out.append(s)
    return out


@pytest.mark.parametrize("scorer", ["WRatio", "QRatio", "partial_ratio", "token_sort_ratio", "token_set_ratio", "token_ratio",
                                    "partial_token_sort_ratio", "partial_token_set_ratio", "partial_token_ratio", "ratio"])
def test_k3b_every_scorer(fz, scorer):
    rng = np.random.default_rng(len(scorer) * 7 + 1)
    frm = _titles(rng, 40) + ["", " ", "The", "a a", "Night of the Living Dead", "x" * 70 + " tail", "long " * 30]
    to = _titles(rng, 120, 1, 9) + ["", "  ", "The", "a", "Dead Night", "x" * 64, "long " * 40, frm[3], frm[3]]
    S = score_matrix(frm, to, scorer)
    for k in KS:
        exp = oracle_topk(S, k, 0.0)
        for n_splits in (1, 3, None):
            _eq(fz.fuzz_topk(frm, to, k, scorer, n_splits=n_splits), exp)
    bi, bs = fz.fuzz_argbest(frm, to, scorer)
    ti, tv = fz.fuzz_topk(frm, to, 10, scorer)
    np.testing.assert_array_equal(ti[:, 0].cpu().numpy(), bi.cpu().numpy())
    np.testing.assert_array_equal(tv[:, 0].cpu().numpy(), bs.cpu().numpy())


def test_k3b_alphabet_batches(fz):
    big = [chr(0x4E00 + i) + " " + chr(0x4E00 + (i * 7) % 600) + "ab" for i in range(600)]
    to = big[::3] + ["ab", "中 ab"]
    S = score_matrix(big, to, "token_set_ratio")
    _eq(fz.fuzz_topk(big, to, 5, "token_set_ratio"), oracle_topk(S, 5, 0.0))


# ---- ties, cutoffs, self-match, duplicates --------------------------------------------------------------------------------
def test_ties_lowest_indices_first(ed, fz):
    rng = np.random.default_rng(5)
    to = _rand_strings(rng, 500, 8, 20, "abcdefgh")
    pos = np.sort(rng.choice(len(to), 50, replace=False))
    for p in pos:
        to[p] = "the same string"
    frm = ["the same string", "the same strinx"]
    for metric in ("ratio", "norm_lev", "jaro_winkler"):
        i, v = ed.edit_topk(frm, to, 10, metric)
        assert i[0].cpu().numpy().tolist() == pos[:10].tolist()
        _eq((i, v), oracle_topk(score_matrix(frm, to, metric), 10, 0.0))
    i, v = fz.fuzz_topk(frm, to, 10, "WRatio")
    assert i[0].cpu().numpy().tolist() == pos[:10].tolist() and (v[0].cpu().numpy() == 100.0).all()


def test_self_match_cutoff_and_short_rows(ed, fz):
    rng = np.random.default_rng(3)
    s = _rand_strings(rng, 300, 3, 20, "abcdef") + ["dup", "dup", "dup"]
    for metric, cut in (("ratio", 60.0), ("norm_lev", 0.5), ("jaro_winkler", 0.85)):
        S = score_matrix(s, s, metric)
        for k in (3, 32):
            exp = oracle_topk(S, k, cut, exclude_self=True)
            _eq(ed.edit_topk(s, s, k, metric, cut, exclude_self=True), exp)
    S = score_matrix(s, s, "token_set_ratio")
    _eq(fz.fuzz_topk(s, s, 10, "token_set_ratio", 70.0, exclude_self=True), oracle_topk(S, 10, 70.0, exclude_self=True))
    # fewer candidates than k: empty slots (-1, 0.0); the row's own index is never returned, its duplicates are
    few = ["abc", "abd", "abc"]
    i, v = ed.edit_topk(few, few, 5, "ratio", exclude_self=True)
    i = i.cpu().numpy(); v = v.cpu().numpy()
    assert i[0].tolist() == [2, 1, -1, -1, -1] and v[0, 2:].tolist() == [0.0] * 3 and v[0, 0] == 100.0
    i, v = fz.fuzz_topk(few, few, 5, "WRatio", exclude_self=True)
    assert i.cpu().numpy()[2].tolist() == [0, 1, -1, -1, -1] and (v.cpu().numpy()[:, 2:] == 0.0).all()


def test_two_lists_with_duplicates(ed, fz):
    rng = np.random.default_rng(9)
    to = _rand_strings(rng, 200, 3, 12, "abcde")
    to = to + to[:50] + to[10:20]
    frm = _rand_strings(rng, 60, 3, 12, "abcde")
    for metric in ("ratio", "jaro"):
        _eq(ed.edit_topk(frm, to, 12, metric), oracle_topk(score_matrix(frm, to, metric), 12, 0.0))
    _eq(fz.fuzz_topk(frm, to, 12, "partial_ratio", 50.0), oracle_topk(score_matrix(frm, to, "partial_ratio"), 12, 50.0))


def test_to_shards_merge_equals_single_call(ed, fz):
    """Single-GPU emulation of distributed=True: per-shard top-k with its global index base and self shift, merged with
    merge_topk_any; the result equals the one-call result."""
    import torch
    from polyfuzz_b200 import synth
    from polyfuzz_b200.distributed import merge_topk_any, shard_bounds
    s = synth.titles(700, seed=4) + ["Alpha", "Alpha"]
    Q = ed.EditQueries(s)
    for metric, cut in (("ratio", 40.0), ("jaro_winkler", 0.6)):
        whole = ed.edit_topk(s, s, 10, metric, cut, exclude_self=True)
        for G in (2, 3):
            parts = []
            for r in range(G):
                lo, hi = shard_bounds(len(s), G, r)
                parts.append(ed.edit_topk_staged(Q, ed.EditTargets(s[lo:hi]), 10, metric, cut, exclude_self=True, self_shift=-lo,
                                                 to_index_base=lo))
            merged = merge_topk_any(torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts]), 10)
            for a, b in zip(whole, merged):
                np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    whole = fz.fuzz_topk(s[:300], s[:300], 7, "WRatio", 50.0, exclude_self=True)
    parts = []
    for r in range(2):
        lo, hi = shard_bounds(300, 2, r)
        parts.append(fz.fuzz_topk(s[:300], s[lo:hi], 7, "WRatio", 50.0, exclude_self=True, self_shift=-lo, to_index_base=lo))
    merged = merge_topk_any(torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts]), 7)
    for a, b in zip(whole, merged):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())


def test_bad_k_is_rejected_on_the_host(ed, fz):
    for k in (0, 33, 2.5, "3", True):
        with pytest.raises(ValueError, match="1 to 32"):
            ed.edit_topk(["a"], ["b"], k)
        with pytest.raises(ValueError, match="1 to 32"):
            fz.fuzz_topk(["a"], ["b"], k)
    with pytest.raises(ValueError, match="metrics"):
        ed.edit_topk(["a"], ["b"], 3, "lev")


# ---- real data -----------------------------------------------------------------------------------------------------------
def test_real_movie_titles(ed, fz):
    from polyfuzz_b200 import datasets
    data, kind = datasets.load_movie_titles()
    if kind != "real":
        pytest.skip("the movie-title fixture is not present")
    frm, to = data["Netflix"], data["IMDB"]
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    for metric in ("ratio", "norm_lev", "jaro_winkler"):
        bi, bs, _ = ed.edit_argbest_staged(Q, T, metric)
        ti, tv = ed.edit_topk_staged(Q, T, 10, metric)
        np.testing.assert_array_equal(ti[:, 0].cpu().numpy(), bi.cpu().numpy())
        np.testing.assert_array_equal(tv[:, 0].cpu().numpy(), bs.cpu().numpy())
        if metric == "ratio":
            rows = np.sort(np.random.default_rng(0).choice(len(frm), 200, replace=False))
            S = score_matrix([frm[i] for i in rows], to, "ratio")
            exp = oracle_topk(S, 10, 0.0)
            np.testing.assert_array_equal(ti.cpu().numpy()[rows], exp[0])
            np.testing.assert_array_equal(tv.cpu().numpy()[rows], exp[1])
    bi, bs = fz.fuzz_argbest(frm, to, "WRatio")
    ti, tv = fz.fuzz_topk(frm, to, 10, "WRatio")
    np.testing.assert_array_equal(ti[:, 0].cpu().numpy(), bi.cpu().numpy())
    np.testing.assert_array_equal(tv[:, 0].cpu().numpy(), bs.cpu().numpy())


# ---- matcher frames ------------------------------------------------------------------------------------------------------
def test_matcher_frames():
    from polyfuzz_b200 import EditDistance, RapidFuzz
    for scorer in ("WRatio", "ratio", "levenshtein"):
        pd.testing.assert_frame_equal(RapidFuzz(scorer=scorer, top_n=1).match(FROM, TO), RapidFuzz(scorer=scorer).match(FROM, TO))
        got = RapidFuzz(scorer=scorer, top_n=3).match(FROM, TO)
        assert list(got.columns) == ["From", "To", "Similarity", "To_2", "Similarity_2", "To_3", "Similarity_3"]
        top1 = RapidFuzz(scorer=scorer).match(FROM, TO)
        pd.testing.assert_frame_equal(got[["From", "To", "Similarity"]], top1)
        metric = {"WRatio": "WRatio", "ratio": "ratio", "levenshtein": "norm_lev"}[scorer]
        exp_i, exp_v = oracle_topk(score_matrix(FROM, TO, metric), 3, 0.0)
        scale = 1.0 if metric == "norm_lev" else 100.0
        assert got.To_3.tolist() == [TO[j] for j in exp_i[:, 2]] and got.Similarity_3.tolist() == (exp_v[:, 2] / scale).tolist()
    # clipping: 3 distinct to-strings -> at most 3 columns; top_n clipped to 1 is the top-1 frame
    assert list(RapidFuzz(top_n=10).match(FROM, TO).columns)[-1] == "Similarity_3"
    pd.testing.assert_frame_equal(RapidFuzz(top_n=5).match(FROM, ["apple", "apple"]), RapidFuzz().match(FROM, ["apple", "apple"]))
    for scorer in ("ratio", "jaro_winkler", "token_set_ratio"):
        pd.testing.assert_frame_equal(EditDistance(scorer=scorer, top_n=1).match(FROM, TO), EditDistance(scorer=scorer).match(FROM, TO))
        e = EditDistance(scorer=scorer, normalize=False, top_n=3).match(FROM, TO)
        pd.testing.assert_frame_equal(e[["From", "To", "Similarity"]], EditDistance(scorer=scorer, normalize=False).match(FROM, TO))
        n = EditDistance(scorer=scorer, top_n=3).match(FROM, TO)
        raw = e[["Similarity", "Similarity_2", "Similarity_3"]].to_numpy()
        np.testing.assert_array_equal(n[["Similarity", "Similarity_2", "Similarity_3"]].to_numpy(),
                                      (raw - raw.min()) / (raw.max() - raw.min()))
    # self-match, not clipped: 6 rows, 5 candidates each -> the 6th slot is empty
    s = EditDistance(normalize=False, top_n=6).match(FROM)
    assert s.To_6.isna().all() and (s.Similarity_6 == 0.0).all() and not (s.To == s.From).any()


def test_reference_orchestrator_with_top_n():
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference orchestrator) was not built")
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    from oracle import ref_shim
    ref_shim.REFERENCE_ROOT = REF
    ref_shim.install()
    from polyfuzz import PolyFuzz
    from polyfuzz_b200 import TFIDF, EditDistance, RapidFuzz
    model = PolyFuzz(RapidFuzz(top_n=3)).match(FROM, TO)
    m = model.get_matches()
    assert list(m.columns) == ["From", "To", "Similarity", "To_2", "Similarity_2", "To_3", "Similarity_3"]
    pd.testing.assert_frame_equal(m[["From", "To", "Similarity"]], RapidFuzz().match(FROM, TO))
    model.group(model=TFIDF(n_gram_range=(3, 3), min_similarity=0.75), link_min_similarity=0.75)
    assert "Group" in model.get_matches().columns
    model = PolyFuzz(EditDistance(top_n=2, normalize=False)).fit(FROM, TO)
    res = model.transform(TO)
    assert list(res[list(res.keys())[0]].columns) == ["From", "To", "Similarity", "To_2", "Similarity_2"]
