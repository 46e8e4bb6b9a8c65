"""GPU tests of candidate mode: K3 / K3b score each from-row against its own candidate list (pfz_lev_rows and
pfz_fuzz_rows with cand_idx; editdist.edit_cand_topk_staged, fuzzy.fuzz_cand_topk) and RapidFuzz / EditDistance(candidates=TFIDF(...)).

The defining property: a row equals the all-pairs result of the same scorer against the to-strings of its candidate list,
indices mapped back, scores bit for bit.  Checked three ways:
  * every to-index as the candidate list (shuffled per row) == the all-pairs kernels on the same lists;
  * random lists (-1 slots, rows with 0 or 1 candidates, c up to 70, i.e. several passes of 32) == the CPU oracles
    (oracle.native / tests/*_oracle / oracle.fuzz) restricted to each row's set, with the kernels' cutoff rules;
  * edges (every K3 / K3b word class, to-strings over 1 024 code points, several alphabet batches, self-match with i in its
    own list, cutoffs at achievable scores from tests/cutoff_cases.py).
Matcher frames are checked against frames built from the oracle TF-IDF's candidates (oracle.tfidf + oracle.native.spdot_topn),
and against the unmodified reference orchestrator.  Indices and scores are compared with ==."""
import functools
import math
import os

import numpy as np
import pandas as pd
import pytest

import cutoff_cases as cc
import dl_oracle
import jaro_oracle
import lcs_oracle
import osa_oracle
from oracle import fuzz as ofuzz
from oracle import native as onative

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
REF = os.path.join(ROOT, "oracle", "_ref")
NT = os.cpu_count() or 1
KS = (1, 3, 32)
K3_METRICS = ("norm_lev", "ratio", "jaro", "jaro_winkler", "norm_osa", "norm_dl")      # editdist.TOPK_METRICS
RAW_METRICS = ("lev", "indel", "osa", "dl")                                             # arg-best only
K3B = ("WRatio", "QRatio", "partial_ratio", "token_sort_ratio", "token_set_ratio", "token_ratio", "partial_token_sort_ratio",
       "partial_token_set_ratio", "partial_token_ratio")
WORDS = ["The", "of", "and", "a", "Night", "Day", "Love", "Man", "Last", "Story", "Dead", "II", "Return", "King", "night", "é",
         "Noël", "x", "Zorro", "Christmas", "Carol", "day", "man", "House", "Home"]


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


def _dev(a):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.int32)).cuda()


def _rand_strings(rng, n, lo, hi, alpha):
    return ["".join(alpha[i] for i in rng.integers(0, len(alpha), rng.integers(lo, hi + 1))) for _ in range(n)]


def _titles(rng, n, lo=1, hi=6):
    out = []
    for _ in range(n):
        ws = list(rng.choice(WORDS, rng.integers(lo, hi + 1)))
        if rng.random() < 0.15:
            ws.append(ws[0])
        out.append(" ".join(ws))
    return out


def _shuffled_all(rng, n_from, n_to):
    return np.stack([rng.permutation(n_to) for _ in range(n_from)]).astype(np.int32)


def _random_lists(rng, n_from, n_to, c):
    """[n_from, c]: distinct to-indices per row with -1 slots interleaved; row 0 empty, row 1 one candidate, row 2 full."""
    cand = np.full((n_from, c), -1, np.int32)
    for i in range(n_from):
        m = 0 if i == 0 else 1 if i == 1 else min(c, n_to) if i == 2 else int(rng.integers(0, min(c, n_to) + 1))
        slots = rng.choice(c, m, replace=False)
        cand[i, slots] = rng.choice(n_to, m, replace=False)
    return cand


# ---- the CPU oracle: one scorer per metric, with the kernels' cutoff rule --------------------------------------------------
class Oracle:
    """score(i, j) -> the kernel's score of (frm[i], to[j]) or None when the cutoff rejects it."""

    def __init__(self, frm, to, metric, cutoff):
        self.frm, self.to, self.metric, self.c = frm, to, metric, cutoff
        self.D, self.memo = None, {}
        la = np.array([len(s) for s in frm], np.float64)[:, None]
        lb = np.array([len(s) for s in to], np.float64)[None, :]
        if metric in ("lev", "norm_lev", "indel", "ratio"):
            self.D = onative.editdist_matrix(frm, to, "indel" if metric in ("indel", "ratio") else "lev", n_threads=NT)
        elif metric in ("osa", "norm_osa"):
            self.D = osa_oracle.osa_matrix(frm, to, n_threads=NT)
        elif metric in ("dl", "norm_dl"):
            self.D = dl_oracle.dl_matrix(frm, to, n_threads=NT)
        if self.D is not None:
            d = self.D.astype(np.float64)
            with np.errstate(invalid="ignore", divide="ignore"):
                if metric == "ratio":
                    m = la + lb
                    self.ns = np.where(m > 0, 1.0 - d / m, 1.0)
                else:
                    m = np.maximum(la, lb)
                    self.ns = np.where(m > 0, 1.0 - d / m, 1.0)

    def score(self, i, j):
        key = (i, j)
        if key not in self.memo:
            self.memo[key] = self._score(i, j)
        return self.memo[key]

    def _score(self, i, j):
        mt, c = self.metric, self.c
        if mt in ("lev", "indel", "osa", "dl"):
            return -float(self.D[i, j])
        if mt == "ratio":
            ns = self.ns[i, j]
            return ns * 100.0 if (ns >= c / 100.0 and ns * 100.0 >= c) else None
        if mt in ("norm_lev", "norm_osa", "norm_dl"):
            s = self.ns[i, j]
        elif mt in ("jaro", "jaro_winkler"):
            s = jaro_oracle.jaro_pair(self.frm[i], self.to[j], winkler=mt == "jaro_winkler")[0]
        else:
            s = ofuzz.SCORERS[mt](self.frm[i], self.to[j], c)
        return s if s >= c else None

    def topk(self, cand, k, exclude_self=False):
        n = cand.shape[0]
        oi = np.full((n, k), -1, np.int32); ov = np.zeros((n, k))
        for i in range(n):
            got = []
            for j in cand[i]:
                if j < 0 or (exclude_self and j == i):
                    continue
                s = self.score(i, int(j))
                if s is not None:
                    got.append((-s, int(j)))
            got.sort()
            for r, (s, j) in enumerate(got[:k]):
                oi[i, r] = j; ov[i, r] = -s
        return oi, ov


def _cand(ed, fz, metric, frm, to, cand, k, cutoff, exclude_self=False, T=None, Q=None):
    """(idx [n, k], score [n, k]) as host arrays from the candidate entry points."""
    if metric in K3B:
        i, v = fz.fuzz_cand_topk(frm, to, _dev(cand), k, metric, cutoff, exclude_self=exclude_self)
    else:
        Q = Q or ed.EditQueries(frm); T = T or ed.EditTargets(to)
        i, v = ed.edit_cand_topk_staged(Q, T, _dev(cand), k, metric, cutoff, exclude_self=exclude_self)[:2]
    i = i.cpu().numpy(); v = v.cpu().numpy()
    return (i[:, None], v[:, None]) if k == 1 else (i, v)


def _no_cut(metric):
    return float("-inf") if metric in K3_METRICS + RAW_METRICS and metric != "ratio" else 0.0


def _eq(got, exp):
    np.testing.assert_array_equal(got[0], exp[0])
    np.testing.assert_array_equal(got[1], exp[1])


# ---- 1. every to-index as the list == all-pairs ------------------------------------------------------------------------------
def _class_strings(rng, alpha, per=(6, 4, 3, 3, 2, 2, 2)):
    spans = [(0, 12), (20, 40), (50, 70), (90, 140), (200, 300), (500, 600), (900, 1024)]
    frm = []
    for (lo, hi), n in zip(spans, per):
        frm += _rand_strings(rng, n, lo, hi, alpha)
    return frm + ["", "a"]


@pytest.mark.parametrize("metric", K3_METRICS + RAW_METRICS)
def test_k3_all_candidates_equal_all_pairs(ed, metric):
    rng = np.random.default_rng(len(metric) * 13 + 1)
    alpha = "abcdefgh éß中K"
    frm = _class_strings(rng, alpha)
    to = _rand_strings(rng, 90, 0, 80, alpha) + _rand_strings(rng, 6, 200, 1100, alpha) + [frm[3], frm[9][:-1], ""]
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    cand = _dev(_shuffled_all(rng, len(frm), len(to)))
    cut = _no_cut(metric)
    gi, gs, gd = ed.edit_cand_topk_staged(Q, T, cand, 1, metric, cut)
    bi, bs, bd = ed.edit_argbest_staged(Q, T, metric, cut)
    for a, b in ((gi, bi), (gs, bs), (gd, bd)):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    if metric in RAW_METRICS:
        return
    for k in KS[1:]:
        gi, gs = ed.edit_cand_topk_staged(Q, T, cand, k, metric, cut)
        ti, ts = ed.edit_topk_staged(Q, T, k, metric, cut)
        np.testing.assert_array_equal(gi.cpu().numpy(), ti.cpu().numpy())
        np.testing.assert_array_equal(gs.cpu().numpy(), ts.cpu().numpy())
    # self-match: every index including i itself, i excluded by the kernel
    cand = _dev(_shuffled_all(rng, len(frm), len(frm)))
    Qs, Ts = ed.EditQueries(frm), ed.EditTargets(frm)
    for k in (1, 5):
        got = ed.edit_cand_topk_staged(Qs, Ts, cand, k, metric, cut, exclude_self=True)
        exp = (ed.edit_argbest_staged(Qs, Ts, metric, cut, exclude_self=True) if k == 1
               else ed.edit_topk_staged(Qs, Ts, k, metric, cut, exclude_self=True))
        for a, b in zip(got, exp):
            np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())


@pytest.mark.parametrize("scorer", K3B + ("ratio",))
def test_k3b_all_candidates_equal_all_pairs(fz, scorer):
    rng = np.random.default_rng(len(scorer) * 7 + 3)
    frm = (_titles(rng, 40) + ["", " ", "The", "a a", "Night of the Living Dead", "x" * 70 + " tail", "long " * 30,
                               " ".join(_titles(rng, 60))[:1024], "y " * 400 + "z" * 100])
    to = _titles(rng, 110, 1, 9) + ["", "  ", "The", "a", "Dead Night", "x" * 64, "long " * 40, frm[3], " ".join(_titles(rng, 260))]
    cand = _dev(_shuffled_all(rng, len(frm), len(to)))
    bi, bs = fz.fuzz_argbest(frm, to, scorer, 0.0)
    gi, gs = fz.fuzz_cand_topk(frm, to, cand, 1, scorer, 0.0)
    np.testing.assert_array_equal(gi.cpu().numpy(), bi.cpu().numpy())
    np.testing.assert_array_equal(gs.cpu().numpy(), bs.cpu().numpy())
    for k in KS[1:]:
        ti, ts = fz.fuzz_topk(frm, to, k, scorer, 0.0)
        gi, gs = fz.fuzz_cand_topk(frm, to, cand, k, scorer, 0.0)
        np.testing.assert_array_equal(gi.cpu().numpy(), ti.cpu().numpy())
        np.testing.assert_array_equal(gs.cpu().numpy(), ts.cpu().numpy())
    # self-match with a cutoff
    cand = _dev(_shuffled_all(rng, len(frm), len(frm)))
    ti, ts = fz.fuzz_topk(frm, frm, 5, scorer, 40.0, exclude_self=True)
    gi, gs = fz.fuzz_cand_topk(frm, frm, cand, 5, scorer, 40.0, exclude_self=True)
    np.testing.assert_array_equal(gi.cpu().numpy(), ti.cpu().numpy())
    np.testing.assert_array_equal(gs.cpu().numpy(), ts.cpu().numpy())


# ---- 2. random lists == the CPU oracle restricted to each row's set -----------------------------------------------------------
@pytest.mark.parametrize("metric", K3_METRICS + RAW_METRICS)
def test_k3_random_lists_vs_oracle(ed, metric):
    rng = np.random.default_rng(len(metric) * 31 + 5)
    alpha = "abcdef éß中"
    frm = _rand_strings(rng, 50, 0, 20, alpha) + _rand_strings(rng, 10, 30, 140, alpha)
    to = _rand_strings(rng, 150, 0, 24, alpha) + _rand_strings(rng, 20, 30, 160, alpha)
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    cut = _no_cut(metric)
    orc = Oracle(frm, to, metric, cut)
    for c in (1, 31, 33, 70):
        cand = _random_lists(rng, len(frm), len(to), c)
        for k in (KS if metric not in RAW_METRICS else (1,)):
            _eq(_cand(ed, None, metric, frm, to, cand, k, cut, Q=Q, T=T), orc.topk(cand, k))


@pytest.mark.parametrize("scorer", K3B)
def test_k3b_random_lists_vs_oracle(fz, scorer):
    rng = np.random.default_rng(len(scorer) * 17 + 2)
    frm = _titles(rng, 30) + ["", "The", "Night of the Living Dead", "x" * 70 + " tail"]
    to = _titles(rng, 90, 1, 9) + ["", "  ", "The", "Dead Night", frm[3]]
    orc = Oracle(frm, to, scorer, 0.0)
    for c in (1, 33, 70):
        cand = _random_lists(rng, len(frm), len(to), c)
        for k in KS:
            _eq(_cand(None, fz, scorer, frm, to, cand, k, 0.0), orc.topk(cand, k))


# ---- 3. edges ----------------------------------------------------------------------------------------------------------------
EDGE_LENS = (0, 1, 32, 33, 64, 65, 256, 257, 1024)


@pytest.mark.parametrize("metric", K3_METRICS + ("lev", "dl"))
def test_k3_every_word_class_and_long_to_strings(ed, metric):
    rng = np.random.default_rng(len(metric) * 3 + 11)
    alpha = "abcdefgh é中"
    frm = [_rand_strings(rng, 1, L, L, alpha)[0] for L in EDGE_LENS for _ in range(2)]
    to = _rand_strings(rng, 60, 0, 70, alpha) + [_rand_strings(rng, 1, L, L, alpha)[0] for L in (256, 1024, 1025, 1500, 2100)]
    to += [frm[8], frm[16][:1000], frm[-1] + "ab"]
    cut = _no_cut(metric)
    orc = Oracle(frm, to, metric, cut)
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    long_to = np.arange(len(to) - 8, len(to), dtype=np.int32)
    for c in (5, 40):
        cand = _random_lists(rng, len(frm), len(to), c)
        cand[3:, 0] = rng.choice(long_to, len(frm) - 3)                   # a long to-string in (almost) every row
        cand = np.array([_dedup(r) for r in cand])
        for k in (KS if metric not in RAW_METRICS else (1,)):
            _eq(_cand(ed, None, metric, frm, to, cand, k, cut, Q=Q, T=T), orc.topk(cand, k))


def _dedup(row):
    seen, out = set(), []
    for j in row:
        out.append(-1 if j in seen else j)
        if j >= 0:
            seen.add(j)
    return np.array(out, np.int32)


@pytest.mark.parametrize("scorer", ("WRatio", "partial_ratio", "token_set_ratio", "partial_token_ratio"))
def test_k3b_every_word_class_and_long_to_strings(fz, scorer):
    """Long pairs are slow in the Python oracle, so rows here are checked against the all-pairs kernels on each row's own
    to-strings (ascending, so the index key is kept) -- the defining property itself."""
    rng = np.random.default_rng(len(scorer) * 5 + 7)
    word = lambda L: (" ".join(_titles(rng, L // 3 + 1)) + " " + "q" * L)[:L]  # noqa: E731
    frm = [word(L) for L in EDGE_LENS for _ in range(2)]
    to = _titles(rng, 60, 1, 9) + [word(L) for L in (256, 1024, 1025, 1500, 2100)] + [frm[8], frm[16][:1000]]
    cand = _random_lists(rng, len(frm), len(to), 40)
    for k in KS:
        gi, gs = _cand(None, fz, scorer, frm, to, cand, k, 0.0)
        for i in range(len(frm)):
            js = np.sort(cand[i][cand[i] >= 0])
            ei = np.full(k, -1, np.int32); es = np.zeros(k)
            if len(js):
                sub = [to[j] for j in js]
                ri, rs = fz.fuzz_topk([frm[i]], sub, k, scorer, 0.0) if k > 1 else fz.fuzz_argbest([frm[i]], sub, scorer, 0.0)
                ri = ri.cpu().numpy().reshape(-1); rs = rs.cpu().numpy().reshape(-1)
                ei = np.where(ri >= 0, js[np.maximum(ri, 0)], -1); es = rs
            np.testing.assert_array_equal(gi[i], ei)
            np.testing.assert_array_equal(gs[i], es)


def test_alphabet_batches(ed, fz):
    """More than 255 distinct code points over the from-list: several alphabet batches, one pfz_lev_pack each."""
    big = [chr(0x4E00 + i) + chr(0x4E00 + (i * 7) % 600) + "ab" for i in range(600)]
    to = big[::3] + ["ab", "中ab"]
    rng = np.random.default_rng(8)
    cand = _random_lists(rng, len(big), len(to), 40)
    for metric in ("norm_lev", "ratio", "jaro_winkler", "norm_osa"):
        orc = Oracle(big, to, metric, 0.0)
        for k in (1, 3):
            _eq(_cand(ed, None, metric, big, to, cand, k, 0.0), orc.topk(cand, k))
    spaced = [s[0] + " " + s[1:] for s in big]
    sto = spaced[::3] + ["ab", "中 ab"]
    orc = Oracle(spaced, sto, "token_set_ratio", 0.0)
    _eq(_cand(None, fz, "token_set_ratio", spaced, sto, cand, 5, 0.0), orc.topk(cand, 5))


def test_self_match_with_i_in_its_own_list(ed, fz):
    rng = np.random.default_rng(4)
    s = _rand_strings(rng, 120, 3, 20, "abcdef") + ["dup", "dup", "dup"]
    cand = _random_lists(rng, len(s), len(s), 20)
    for i in range(len(s)):                                            # i is in its own list, at a random slot
        if i not in cand[i]:
            cand[i, rng.integers(0, 20)] = i
    cand = np.array([_dedup(r) for r in cand])
    for metric, cut in (("ratio", 50.0), ("norm_lev", 0.4), ("jaro_winkler", 0.8), ("norm_dl", 0.3)):
        orc = Oracle(s, s, metric, cut)
        for k in KS:
            got = _cand(ed, None, metric, s, s, cand, k, cut, exclude_self=True)
            _eq(got, orc.topk(cand, k, exclude_self=True))
            assert not (got[0] == np.arange(len(s))[:, None]).any()
    orc = Oracle(s, s, "WRatio", 60.0)
    for k in (1, 5):
        _eq(_cand(None, fz, "WRatio", s, s, cand, k, 60.0, exclude_self=True), orc.topk(cand, k, exclude_self=True))


def test_cutoffs_at_achievable_scores(ed, fz):
    """ratio and the partial scorers at their boundary pairs (a cutoff equal to the pair's own score rejects it), and the 0..1
    metrics at achieved scores (kept) and one ulp above (rejected)."""
    rng = np.random.default_rng(12)
    filler = _rand_strings(rng, 40, 1, 30, "abc ")
    trip = [t for t in cc.ratio_triples(30) if cc.is_boundary_score(cc.ratio_ns(*t))][:: 97][:6]
    for la, lb, lcs in trip:
        a, b = cc.ratio_strings(la, lb, lcs)
        s = cc.ratio_ns(la, lb, lcs) * 100.0
        to = filler + [b]
        cand = np.array([[len(to) - 1] + list(rng.choice(len(filler), 9, replace=False))], np.int32)
        for c in cc.neighbours(s):
            orc = Oracle([a], to, "ratio", c)
            for k in (1, 3):
                _eq(_cand(ed, None, "ratio", [a], to, cand, k, c), orc.topk(cand, k))
        assert _cand(ed, None, "ratio", [a], to, cand, 1, s)[0][0, 0] != len(to) - 1
    for scorer in ("partial_ratio", "WRatio", "token_ratio"):
        for a, b, s in cc.boundary_pairs(scorer, 3, seed=len(scorer)):
            to = filler + [b]
            cand = np.array([[len(to) - 1] + list(rng.choice(len(filler), 9, replace=False))], np.int32)
            for c in cc.neighbours(s):
                orc = Oracle([a], to, scorer, c)
                for k in (1, 3):
                    _eq(_cand(None, fz, scorer, [a], to, cand, k, c), orc.topk(cand, k))
    frm = _rand_strings(rng, 20, 2, 12, "abcd")
    to = _rand_strings(rng, 60, 2, 12, "abcd")
    cand = _random_lists(rng, len(frm), len(to), 12)
    for metric in ("norm_lev", "jaro", "norm_osa", "norm_dl"):
        free = Oracle(frm, to, metric, float("-inf"))
        for i in (2, 5):
            j = int(cand[i][cand[i] >= 0][0])
            s = free.score(i, j)
            for c in (s, math.nextafter(s, math.inf)):
                orc = Oracle(frm, to, metric, c)
                for k in (1, 3):
                    _eq(_cand(ed, None, metric, frm, to, cand, k, c), orc.topk(cand, k))


def test_matrix_and_gate_of_lev_rows_in_candidate_mode(ed):
    """pfz_lev_rows in candidate mode with k = 0 and a matrix: the candidate pairs' cells hold their distances, the rest is
    untouched; with dl and a gate (each row's best OSA score over its list) it returns the ungated result."""
    import torch
    from polyfuzz_b200 import _lib
    from polyfuzz_b200.engine import _p, _stream
    rng = np.random.default_rng(21)
    frm = _rand_strings(rng, 30, 0, 70, "abcde")
    to = _rand_strings(rng, 80, 0, 70, "abcde")
    cand = _random_lists(rng, len(frm), len(to), 20)
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    dc = _dev(cand)

    def rows(metric, mat, gate):
        out = [torch.full((len(frm),), -1, dtype=torch.int32, device="cuda"), torch.zeros(len(frm), dtype=torch.float64, device="cuda"),
               torch.full((len(frm),), -1, dtype=torch.int32, device="cuda")]
        counter = torch.zeros(1, dtype=torch.int32, device="cuda")
        for d_table, nw, d_ids, n_ids in ed._word_classes(Q, T):
            _lib.call("pfz_lev_rows", _p(Q.d_blob), _p(Q.d_off), Q.n, _p(d_ids), n_ids, nw, _p(d_table), _p(T.packed), _p(T.d_goff),
                      _p(T.slen), _p(T.d_order), T.n, ed.METRIC[metric], 0.0, 0, 0, 1, 0, _p(dc), cand.shape[1], _p(T.d_pos_of),
                      *[_p(t) for t in out], _p(mat), int(mat.stride(0)) if mat is not None else 0, _p(gate), _p(counter), _stream())
        return out

    for metric, D in (("lev", onative.editdist_matrix(frm, to, "lev")), ("osa", osa_oracle.osa_matrix(frm, to)),
                      ("dl", dl_oracle.dl_matrix(frm, to))):
        mat = torch.full((len(frm), len(to)), -7, dtype=torch.int32, device="cuda")
        out = rows(metric, mat, None)
        m = mat.cpu().numpy()
        exp = np.full_like(m, -7)
        for i in range(len(frm)):
            js = cand[i][cand[i] >= 0]
            exp[i, js] = D[i, js]
        np.testing.assert_array_equal(m, exp)
        ref = ed.edit_cand_topk_staged(Q, T, dc, 1, metric, 0.0)
        for a, b in zip(out, ref):
            np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    # the gate: the best norm_osa score over each row's list bounds its best norm_dl score from below
    oi, os_, _ = ed.edit_cand_topk_staged(Q, T, dc, 1, "norm_osa", 0.0)
    gate = torch.where(oi >= 0, os_, 0.0).contiguous()
    out = rows("norm_dl", None, gate)
    ref = ed.edit_cand_topk_staged(Q, T, dc, 1, "norm_dl", 0.0)
    for a, b in zip(out[:2], ref[:2]):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())


def test_bad_candidate_arrays_are_refused(ed, fz):
    import torch
    Q, T = ed.EditQueries(["ab", "cd"]), ed.EditTargets(["ab", "x", "cd"])
    good = _dev([[0, -1], [2, 1]])
    for bad in (good.cpu(), good.long(), good[:1], _dev([[0, 3], [1, 2]]), _dev([[-2, 0], [1, 2]]), torch.zeros(2, device="cuda")):
        with pytest.raises(ValueError):
            ed.edit_cand_topk_staged(Q, T, bad, 1, "ratio")
        with pytest.raises(ValueError):
            fz.fuzz_cand_topk(["ab", "cd"], ["ab", "x", "cd"], bad, 2, "WRatio")
    with pytest.raises(ValueError, match="metrics"):
        ed.edit_cand_topk_staged(Q, T, good, 2, "lev")
    # no candidates at all: every slot empty
    i, s, d = ed.edit_cand_topk_staged(Q, T, _dev(np.zeros((2, 0))), 1, "ratio")
    assert i.tolist() == [-1, -1] and s.tolist() == [0.0, 0.0] and d.tolist() == [-1, -1]
    i, s = fz.fuzz_cand_topk(["ab", "cd"], ["ab", "x", "cd"], _dev(-np.ones((2, 4))), 3, "WRatio")
    assert (i.cpu().numpy() == -1).all() and (s.cpu().numpy() == 0.0).all()


# ---- 4. matchers on the golden slices ---------------------------------------------------------------------------------------
def _oracle_cands(frm, to, c):
    """The oracle TF-IDF's top-c (min_similarity 0, sparse): to_list None is a self-match."""
    from oracle import tfidf
    f, t, _ = tfidf.fit_transform_sklearn(frm, to)
    return onative.spdot_topn(f, t, c, 0.0, self_match=to is None, n_threads=NT)[0]


def _oracle_frame(frm, targets, orc, cand, k, scale, exclude_self):
    oi, ov = orc.topk(cand, k, exclude_self)
    cols = {"From": pd.Series(list(frm), dtype=object)}
    for r in range(k):
        cols["To" if r == 0 else f"To_{r + 1}"] = pd.Series([targets[j] if j >= 0 else None for j in oi[:, r]], dtype=object)
        cols["Similarity" if r == 0 else f"Similarity_{r + 1}"] = np.where(oi[:, r] >= 0, ov[:, r] / scale, 0.0)
    return pd.DataFrame(cols), oi


def test_matchers_on_the_company_slice(golden_dir):
    import json
    from polyfuzz_b200 import TFIDF, EditDistance, RapidFuzz
    names = json.load(open(os.path.join(golden_dir, "company_slice_names.json")))["names"][:1000]
    c = 10
    cand = _oracle_cands(names, None, c)
    np.testing.assert_array_equal(TFIDF(top_n=c, min_similarity=0).match_arrays(names)[0].cpu().numpy(), cand)
    wratio = Oracle(names, names, "WRatio", 0.0)
    for top_n in (1, 3):
        got = RapidFuzz(top_n=top_n, candidates=TFIDF(top_n=c, min_similarity=0)).match(names)
        exp, oi = _oracle_frame(names, names, wratio, cand, top_n, 100.0, True)
        pd.testing.assert_frame_equal(got, exp)
        assert (oi[:, 0] >= 0).sum() > 900
    got = RapidFuzz(scorer="ratio", score_cutoff=0.6, top_n=2, candidates=TFIDF(top_n=c, min_similarity=0)).match(names)
    exp, _ = _oracle_frame(names, names, Oracle(names, names, "ratio", 60.0), cand, 2, 100.0, True)
    pd.testing.assert_frame_equal(got, exp)
    got = EditDistance(scorer="levenshtein", normalize=False, candidates=TFIDF(top_n=c, min_similarity=0)).match(names)
    exp, _ = _oracle_frame(names, names, Oracle(names, names, "norm_lev", float("-inf")), cand, 1, 1.0, True)
    pd.testing.assert_frame_equal(got, exp)


def test_matchers_on_the_titles_slice(golden_dir):
    import json
    from polyfuzz_b200 import TFIDF, EditDistance, RapidFuzz
    g = json.load(open(os.path.join(golden_dir, "titles_slice_names.json")))
    frm, to = g["from"], g["to"]
    c = 20
    cand = _oracle_cands(frm, to, c)
    np.testing.assert_array_equal(TFIDF(top_n=c, min_similarity=0).match_arrays(frm, to)[0].cpu().numpy(), cand)
    got = RapidFuzz(top_n=3, candidates=TFIDF(top_n=c, min_similarity=0)).match(frm, to)
    exp, _ = _oracle_frame(frm, to, Oracle(frm, to, "WRatio", 0.0), cand, 3, 100.0, False)
    pd.testing.assert_frame_equal(got, exp)
    for scorer, metric, normalize in (("ratio", "ratio", False), ("jaro_winkler", "jaro_winkler", True), ("osa", "norm_osa", True),
                                      ("token_sort_ratio", "token_sort_ratio", False)):
        got = EditDistance(scorer=scorer, top_n=2, normalize=normalize, candidates=TFIDF(top_n=c, min_similarity=0)).match(frm, to)
        orc = Oracle(frm, to, metric, 0.0 if metric in K3B else float("-inf"))
        exp, oi = _oracle_frame(frm, to, orc, cand, 2, 1.0, False)
        if normalize:
            s = exp[["Similarity", "Similarity_2"]].to_numpy()
            filled = oi >= 0
            lo, hi = s[filled].min(), s[filled].max()
            exp[["Similarity", "Similarity_2"]] = np.where(filled, (s - lo) / (hi - lo), 0.0)
        pd.testing.assert_frame_equal(got, exp)


# ---- 5. through the unmodified orchestrator -------------------------------------------------------------------------------
def test_reference_orchestrator_fit_transform_and_joblib(tmp_path):
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference orchestrator) was not built")
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    from oracle import ref_shim
    ref_shim.REFERENCE_ROOT = REF
    ref_shim.install()
    from polyfuzz import PolyFuzz
    from polyfuzz_b200 import TFIDF, EditDistance, RapidFuzz, synth
    to = list(dict.fromkeys(synth.company_names(300, seed=31)))          # distinct: TF-IDF's top_n is clipped to len(set(to))
    new = synth.company_names(120, seed=32) + to[:10]
    # top_n of the TF-IDF >= len(to): a row's list is every to-string sharing an n-gram with it, whichever list the
    # vectoriser was fitted on, so transform() equals a fresh match(new, to)
    makers = [lambda: RapidFuzz(top_n=3, candidates=TFIDF(top_n=len(to), min_similarity=0)),
              lambda: RapidFuzz(scorer="ratio", candidates=TFIDF(top_n=len(to), min_similarity=0)),
              lambda: EditDistance(scorer="jaro_winkler", top_n=2, candidates=TFIDF(top_n=len(to), min_similarity=0))]
    for mk in makers:
        model = PolyFuzz(mk()).fit(to)
        res = model.transform(new)
        got = res[list(res.keys())[0]]
        pd.testing.assert_frame_equal(got, mk().match(new, to))
        pd.testing.assert_frame_equal(model.transform(new)[list(res.keys())[0]], got)           # kept to-side and index
        path = str(tmp_path / "pf.joblib")
        model.save(path)
        loaded = PolyFuzz.load(path)
        pd.testing.assert_frame_equal(loaded.transform(new)[list(res.keys())[0]], got)
    # fit(from, to) then match through PolyFuzz.match
    m = PolyFuzz(RapidFuzz(top_n=2, candidates=TFIDF(top_n=5, min_similarity=0))).match(new, to).get_matches()
    assert list(m.columns) == ["From", "To", "Similarity", "To_2", "Similarity_2"]
    pd.testing.assert_frame_equal(m, RapidFuzz(top_n=2, candidates=TFIDF(top_n=5, min_similarity=0)).match(new, to))
