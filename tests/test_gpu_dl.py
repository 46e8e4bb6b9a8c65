"""GPU parity tests of the unrestricted Damerau-Levenshtein mode of K3 (csrc/pfz_lev.cu, dl_kernel: an OSA gate, OSA bounds and
a queued exact DP) against the full-matrix Lowrance-Wagner DP of the CPU oracle (tests/dl_oracle.c).  Indices, scores, distances
and matrices are compared with ==: the kernel's score is the same IEEE expression as the oracle's."""
import os

import numpy as np
import pytest

import dl_oracle
import osa_oracle

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
REF = os.path.join(ROOT, "oracle", "_ref")
NT = os.cpu_count() or 1
METRICS = ["norm_dl", "dl"]
KS = [2, 3, 10, 31, 32]


@pytest.fixture(scope="module")
def ed():
    from polyfuzz_b200 import editdist
    return editdist


def _rand_strings(rng, n, lo, hi, alpha):
    return ["".join(alpha[i] for i in rng.integers(0, len(alpha), rng.integers(lo, hi + 1))) for _ in range(n)]


def _swap_gap(s, p, ins="z"):
    """s with s[p] and s[p + 1] exchanged and `ins` put between them: dl = 2, osa = 3 when the two characters differ."""
    return s[:p] + s[p + 1] + ins + s[p] + s[p + 2:] if p + 1 < len(s) else s


def _check(ed, frm, to, metric, score_cutoff=0.0, exclude_self=False, n_splits=None, matrix=False, dl_gate=True):
    got = ed.edit_argbest(frm, to, metric, score_cutoff=score_cutoff, exclude_self=exclude_self, want_matrix=matrix,
                          n_splits=n_splits, dl_gate=dl_gate)
    oi, os_, od = dl_oracle.dl_argbest(frm, to, metric, score_cutoff=score_cutoff, exclude_self=exclude_self, n_threads=NT)
    np.testing.assert_array_equal(got[0].cpu().numpy(), oi)
    np.testing.assert_array_equal(got[1].cpu().numpy(), os_)
    np.testing.assert_array_equal(got[2].cpu().numpy(), od)
    if matrix:
        np.testing.assert_array_equal(got[3].cpu().numpy(), dl_oracle.dl_matrix(frm, to, n_threads=NT))
    return oi, os_, od


def score_matrix(frm, to):
    """float64 [n_from, n_to] of norm_dl, the kernel's expression on the oracle's distances."""
    d = dl_oracle.dl_matrix(frm, to, n_threads=NT).astype(np.float64)
    m = np.maximum(np.array([len(s) for s in frm], dtype=np.float64)[:, None], np.array([len(s) for s in to], dtype=np.float64)[None, :])
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(m > 0, 1.0 - d / m, 1.0)


def oracle_topk(S, k, cutoff=float("-inf"), exclude_self=False):
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


def _check_topk(ed, Q, T, S, k, cutoff=0.0, exclude_self=False, n_splits=None, dl_gate=True):
    got = ed.edit_topk_staged(Q, T, k, "norm_dl", cutoff, exclude_self=exclude_self, n_splits=n_splits, dl_gate=dl_gate)
    exp = oracle_topk(S, k, cutoff, exclude_self)
    np.testing.assert_array_equal(got[0].cpu().numpy(), exp[0])
    np.testing.assert_array_equal(got[1].cpu().numpy(), exp[1])


CLASSES = [(0, 12, 70, 200), (20, 40, 70, 150), (50, 70, 60, 120), (90, 140, 40, 100), (200, 300, 24, 60), (500, 600, 12, 40),
           (900, 1024, 8, 24)]


def _class_lists(lo, hi, n_from, n_to, seed):
    rng = np.random.default_rng(seed)
    alpha = "abcdefgh éß中K"
    frm = _rand_strings(rng, n_from, lo, hi, alpha) + ["", "a"]
    near = [_swap_gap(frm[r], int(rng.integers(0, max(1, len(frm[r]) - 1)))) for r in range(0, n_from, 5)]
    to = _rand_strings(rng, n_to, max(0, lo // 2), hi + 10, alpha) + ["", frm[3], frm[3][:-1] if frm[3] else "x"] + near
    return frm, to


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("lo,hi,n_from,n_to", CLASSES)
def test_every_word_class_with_matrix(ed, metric, lo, hi, n_from, n_to):
    frm, to = _class_lists(lo, hi, n_from, n_to, lo * 7 + hi + 1)
    for n_splits in (1, 3, None):
        _check(ed, frm, to, metric, n_splits=n_splits, matrix=True)
        _check(ed, frm, to, metric, n_splits=n_splits)
    _check(ed, frm, to, metric, dl_gate=False)


@pytest.mark.parametrize("lo,hi,n_from,n_to", CLASSES)
def test_topk_every_word_class(ed, lo, hi, n_from, n_to):
    frm, to = _class_lists(lo, hi, n_from, n_to, lo * 3 + hi)
    S = score_matrix(frm, to)
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    for k in KS:
        for n_splits in (1, 3, None):
            _check_topk(ed, Q, T, S, k, n_splits=n_splits)
    _check_topk(ed, Q, T, S, 10, dl_gate=False)
    bi, bs, _ = ed.edit_argbest_staged(Q, T, "norm_dl", 0.0)
    ti, tv = ed.edit_topk_staged(Q, T, 10, "norm_dl", 0.0)
    np.testing.assert_array_equal(ti[:, 0].cpu().numpy(), bi.cpu().numpy())
    np.testing.assert_array_equal(tv[:, 0].cpu().numpy(), bs.cpu().numpy())


@pytest.mark.parametrize("metric", METRICS)
def test_dl_below_osa_at_word_and_block_edges(ed, metric):
    """A swap with a character inserted between the swapped pair (dl = 2, osa = 3) at pattern positions 31/32, 63/64,
    127/128 and 511/512: the bounds do not meet, so each pair takes the exact DP, across the 32- and 64-bit block edges."""
    rng = np.random.default_rng(7)
    frm, to = [], []
    for length, positions in ((32, (0, 15, 30)), (33, (31,)), (64, (31, 62)), (65, (63,)), (100, (63, 64)), (129, (127,)),
                              (200, (63, 127, 128)), (300, (255, 256)), (700, (511, 600)), (1024, (511, 1022))):
        for p in positions:
            s = "".join(rng.choice(list("abcdefghijklmnop"), length))
            while s[p] == s[p + 1]:
                s = "".join(rng.choice(list("abcdefghijklmnop"), length))
            frm.append(s); to.append(_swap_gap(s, p))
    to = to + _rand_strings(rng, 50, 20, 300, "abcdefghijklmnop")
    oi, _, od = _check(ed, frm, to, metric, matrix=True)
    assert (od == 2).all() and (oi == np.arange(len(frm))).all()
    assert (np.diag(osa_oracle.osa_matrix(frm, to[:len(frm)], n_threads=NT)) == 3).all()
    _check(ed, frm, to, metric)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("alpha", ["ab", "abc"])
def test_tiny_alphabets_non_ascii_text_only_and_empty(ed, metric, alpha):
    rng = np.random.default_rng(len(alpha) + 40)
    frm = _rand_strings(rng, 150, 0, 40, alpha) + _rand_strings(rng, 20, 60, 130, alpha) + ["", "é", "中ab", "ß" * 33, "ba", "CA"]
    # "xyzXYZ" and "ABC" hold code points no from-string has: they map to symbol 0, which matches nothing
    to = _rand_strings(rng, 400, 0, 60, alpha) + ["", "é", "ab中", "xyzXYZ", "ß" * 20, "ab", "ABC", "aXb", "bXa"]
    _check(ed, frm, to, metric, matrix=True)
    _check(ed, frm, to, metric, n_splits=3)
    if metric == "norm_dl":
        S = score_matrix(frm, to)
        Q, T = ed.EditQueries(frm), ed.EditTargets(to)
        for k in (3, 32):
            _check_topk(ed, Q, T, S, k)


def test_alphabet_batches(ed):
    big = [chr(0x4E00 + i) + chr(0x4E00 + (i * 7) % 600) + "abc" for i in range(600)]
    to = big[::3] + ["ab", "中ab"] + [s[1] + "x" + s[0] + s[2:] for s in big[1::7]]
    assert len(set("".join(big))) > 255
    for metric in METRICS:
        _check(ed, big, to, metric, matrix=True)
        _check(ed, big, to, metric)
    _check_topk(ed, ed.EditQueries(big), ed.EditTargets(to), score_matrix(big, to), 5)


def test_self_match_with_and_without_cutoff(ed):
    rng = np.random.default_rng(3)
    s = _rand_strings(rng, 400, 3, 20, "abcdef") + ["dup", "dup", "dpu"]
    for metric, cut in (("norm_dl", 0.0), ("norm_dl", 0.8), ("dl", 0.9)):
        oi, _, _ = _check(ed, s, s, metric, score_cutoff=cut, exclude_self=True)
        assert (oi != np.arange(len(s))).all() and oi[-3] == len(s) - 2 and oi[-2] == len(s) - 3
        if metric == "norm_dl" and cut == 0.8:
            assert (oi == -1).any()
    S = score_matrix(s, s)
    Q = ed.EditQueries(s); T = ed.EditTargets(s)
    for k in (3, 32):
        for cut in (0.0, 0.7):
            _check_topk(ed, Q, T, S, k, cutoff=cut, exclude_self=True)


def test_heavy_ties_and_duplicates(ed):
    """600 identical rows pin every gate at 1.0 and fill the queue; the canonical key must still pick the lowest indices."""
    dup = ["abcdef"] * 600 + ["abdcef", "bacdef", "abcfed", "acbdxef"]
    frm = ["abcdef", "abdcef", "acbdef", "fedcba", "abc"]
    _check(ed, frm, dup, "norm_dl")
    _check(ed, frm, dup, "dl")
    _check(ed, dup[:40] + dup[600:], dup, "norm_dl", exclude_self=True)
    S = score_matrix(frm, dup)
    Q, T = ed.EditQueries(frm), ed.EditTargets(dup)
    for k in KS:
        for n_splits in (1, 3, None):
            _check_topk(ed, Q, T, S, k, n_splits=n_splits)


def test_rows_with_fewer_than_k_candidates(ed):
    frm = ["abcd", "zzzz", "", "dcba"]
    to = ["abdc", "abcx", "bacd", "qqqq", "ab"]
    S = score_matrix(frm, to)
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    for k in (3, 10, 32):
        for cut in (0.0, 0.5, 0.75):
            _check_topk(ed, Q, T, S, k, cutoff=cut)
    with pytest.raises(ValueError, match="top-k"):
        ed.edit_topk(["ab"], ["ba"], 2, "dl")


def test_to_shards_merge_equals_single_call(ed):
    """Single-GPU emulation of distributed=True: each to-shard staged and gated separately, with its global index base and
    self shift; arg-best merged by lev_merge, top-k by merge_topk_any."""
    import torch
    from polyfuzz_b200 import synth
    from polyfuzz_b200.distributed import merge_topk_any, shard_bounds
    s = synth.titles(700, seed=4) + ["Alpha", "Alpha", "lApha", "lpAha"]
    whole = ed.edit_argbest(s, s, "norm_dl", score_cutoff=0.6, exclude_self=True)
    Q = ed.EditQueries(s)
    parts, tparts = [], []
    for r in range(2):
        lo, hi = shard_bounds(len(s), 2, r)
        T = ed.EditTargets(s[lo:hi])
        parts.append(ed.edit_argbest_staged(Q, T, "norm_dl", 0.6, exclude_self=True, self_shift=-lo, to_index_base=lo))
        tparts.append(ed.edit_topk_staged(Q, T, 5, "norm_dl", 0.6, exclude_self=True, self_shift=-lo, to_index_base=lo))
    merged = ed.lev_merge(*(torch.stack([p[c] for p in parts]) for c in range(3)))
    for a, b in zip(whole, merged):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    oi, os_, od = dl_oracle.dl_argbest(s, s, "norm_dl", score_cutoff=0.6, exclude_self=True, n_threads=NT)
    np.testing.assert_array_equal(merged[0].cpu().numpy(), oi); np.testing.assert_array_equal(merged[1].cpu().numpy(), os_)
    np.testing.assert_array_equal(merged[2].cpu().numpy(), od)
    mi, mv = merge_topk_any(torch.stack([t[0] for t in tparts]), torch.stack([t[1] for t in tparts]), 5)
    exp = oracle_topk(score_matrix(s, s), 5, 0.6, exclude_self=True)
    np.testing.assert_array_equal(mi.cpu().numpy(), exp[0]); np.testing.assert_array_equal(mv.cpu().numpy(), exp[1])


FROM = ["CA", "Jhon Smtih", "Micorsoft", "apple", "appel", "house", "similarity"]
TO = ["ABC", "XY", "Joan Smyth", "John Smith", "Microsoft", "apple", "apples", "mouse"]


def test_issue_example_dl_against_osa():
    from polyfuzz_b200 import EditDistance
    got = EditDistance(scorer="dl", normalize=False).match(["CA"], ["ABC", "XY"])
    assert got.To.tolist() == ["ABC"] and got.Similarity.tolist() == [1.0 - 2 / 3]
    got = EditDistance(scorer="osa", normalize=False).match(["CA"], ["ABC", "XY"])
    assert got.Similarity.tolist() == [0.0]


@pytest.mark.parametrize("normalize", [True, False])
def test_editdistance_frames(normalize):
    from polyfuzz_b200 import EditDistance
    got = EditDistance(n_jobs=1, scorer="dl", normalize=normalize).match(FROM, TO)
    oi, os_, _ = dl_oracle.dl_argbest(FROM, TO, "norm_dl", score_cutoff=float("-inf"))
    assert got.From.tolist() == FROM and got.To.tolist() == [TO[i] for i in oi]
    exp = os_ if not normalize else (os_ - os_.min()) / (os_.max() - os_.min())
    np.testing.assert_array_equal(got.Similarity.to_numpy(), exp)
    got = EditDistance(scorer="dl", normalize=False).match(FROM + ["apple"])          # self-match excludes index i only
    oi, os_, _ = dl_oracle.dl_argbest(FROM + ["apple"], FROM + ["apple"], "norm_dl", score_cutoff=float("-inf"), exclude_self=True)
    assert got.To.tolist() == [(FROM + ["apple"])[i] for i in oi] and got.Similarity.tolist() == os_.tolist()


def test_rapidfuzz_top3_frame():
    from polyfuzz_b200 import RapidFuzz
    df = RapidFuzz(scorer="dl", score_cutoff=0.8, top_n=3).match(FROM, TO)
    exp_i, exp_v = oracle_topk(score_matrix(FROM, TO), 3, 0.8)
    for r, (tc, sc) in enumerate((("To", "Similarity"), ("To_2", "Similarity_2"), ("To_3", "Similarity_3"))):
        assert df[tc].tolist() == [TO[j] if j >= 0 else None for j in exp_i[:, r]]
        assert df[sc].tolist() == [v if j >= 0 else 0.0 for v, j in zip(exp_v[:, r], exp_i[:, r])]
    df = RapidFuzz(scorer="dl", score_cutoff=0.3).match(FROM, TO)
    oi, os_, _ = dl_oracle.dl_argbest(FROM, TO, "norm_dl", score_cutoff=0.3)
    assert df.To.tolist() == [TO[i] if i >= 0 else None for i in oi] and df.Similarity.tolist() == os_.tolist()


def test_real_movie_titles_sample(ed):
    from polyfuzz_b200 import datasets
    data, kind = datasets.load_movie_titles()
    if kind != "real":
        pytest.skip("the movie-title fixture is not present")
    rng = np.random.default_rng(0)
    rows = np.sort(rng.choice(len(data["Netflix"]), 300, replace=False))
    frm = [data["Netflix"][i] for i in rows]
    _check(ed, frm, data["IMDB"], "norm_dl")
    Q, T = ed.EditQueries(frm[:60]), ed.EditTargets(data["IMDB"])
    _check_topk(ed, Q, T, score_matrix(frm[:60], data["IMDB"]), 10)


SNIPPET = """
from polyfuzz import PolyFuzz
from polyfuzz.models import EditDistance

from_list = ["CA", "Jhon Smtih", "Micorsoft", "apple", "appel", "house", "similarity"]
to_list = ["ABC", "XY", "Joan Smyth", "John Smith", "Microsoft", "apple", "apples", "mouse"]

model = PolyFuzz(EditDistance(n_jobs=1, scorer=SCORER)).match(from_list, to_list)
"""


def test_reference_orchestrator(monkeypatch):
    """PolyFuzz(EditDistance(scorer=...)) through the unmodified reference orchestrator: first with the reference's own
    EditDistance calling a stand-in DL scorer (the CPU oracle, named like rapidfuzz's), then after polyfuzz_b200.install(),
    which puts this package's EditDistance behind the same names.  Both frames must be equal."""
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference orchestrator) was not built")
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    from oracle import ref_shim
    ref_shim.REFERENCE_ROOT = REF
    ref_shim.install()

    def damerau_levenshtein_normalized_similarity(s1, s2):
        return dl_oracle.norm_dl(s1, s2)

    import polyfuzz.models as pm
    import polyfuzz.polyfuzz as pp
    for mod in (pm, pp):                                   # install() rebinds these; undone after the test
        for name in ("TFIDF", "RapidFuzz", "EditDistance", "Embeddings"):
            if hasattr(mod, name):
                monkeypatch.setattr(mod, name, getattr(mod, name))
    ns_ref = {"SCORER": damerau_levenshtein_normalized_similarity}
    exec(SNIPPET, ns_ref)
    ref = ns_ref["model"].get_matches()
    import polyfuzz_b200
    polyfuzz_b200.install()
    ns_gpu = {"SCORER": damerau_levenshtein_normalized_similarity}
    exec(SNIPPET, ns_gpu)
    got = ns_gpu["model"].get_matches()
    assert list(got.columns) == list(ref.columns) == ["From", "To", "Similarity"]
    assert got.From.tolist() == ref.From.tolist() and got.To.tolist() == ref.To.tolist()
    assert got.To.tolist()[:3] == ["ABC", "John Smith", "Microsoft"]
    np.testing.assert_array_equal(got.Similarity.to_numpy(dtype=np.float64), ref.Similarity.to_numpy(dtype=np.float64))
