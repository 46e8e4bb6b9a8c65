"""GPU parity tests of the Jaro / Jaro-Winkler mode of K3 (csrc/pfz_lev.cu, text-driven bit-parallel matching) against
the pattern-driven CPU oracle (tests/jaro_oracle.c).  Indices, scores and match counts are compared with ==: the kernel
evaluates the definition's float64 expression in the same order with the same roundings."""
import os
import sys

import numpy as np
import pytest

import jaro_oracle

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
REF = os.path.join(ROOT, "oracle", "_ref")
FROM = ["apple", "apples", "appl", "recal", "house", "similarity"]
TO = ["apple", "apples", "mouse"]
METRICS = ["jaro", "jaro_winkler"]
NT = os.cpu_count() or 1


@pytest.fixture(scope="module")
def ed():
    from polyfuzz_b200 import editdist
    return editdist


def _rand_strings(rng, n, lo, hi, alpha):
    return ["".join(alpha[i] for i in rng.integers(0, len(alpha), rng.integers(lo, hi + 1))) for _ in range(n)]


def _check(ed, frm, to, metric, score_cutoff=float("-inf"), exclude_self=False, n_splits=None):
    bi, bs, bd = ed.edit_argbest(frm, to, metric, score_cutoff=score_cutoff, exclude_self=exclude_self, n_splits=n_splits)
    oi, os_, od = jaro_oracle.jaro_argbest(frm, to, metric, score_cutoff=score_cutoff, exclude_self=exclude_self, n_threads=NT)
    np.testing.assert_array_equal(bi.cpu().numpy(), oi)
    np.testing.assert_array_equal(bd.cpu().numpy(), od)
    np.testing.assert_array_equal(bs.cpu().numpy(), os_)
    return oi, os_, od


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("lo,hi,n_from,n_to", [(0, 12, 70, 200), (20, 40, 70, 150), (50, 70, 60, 120), (90, 140, 40, 100),
                                               (200, 300, 24, 60), (500, 600, 12, 40), (900, 1024, 8, 24)])
def test_random_strings_all_word_classes(ed, metric, lo, hi, n_from, n_to):
    rng = np.random.default_rng(lo * 7 + hi)
    alpha = "abcdefgh éß中K"
    frm = _rand_strings(rng, n_from, lo, hi, alpha) + ["", "a"]
    to = _rand_strings(rng, n_to, max(0, lo // 2), hi + 10, alpha) + ["", frm[3], frm[3][:-1] if frm[3] else "x", frm[4][::-1]]
    _check(ed, frm, to, metric, n_splits=3)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("alpha", ["ab", "abc"])
def test_tiny_alphabets_ties_non_ascii_and_empty(ed, metric, alpha):
    rng = np.random.default_rng(len(alpha))
    frm = _rand_strings(rng, 150, 0, 40, alpha) + _rand_strings(rng, 20, 60, 130, alpha) + ["", "é", "中ab", "ß" * 33]
    to = _rand_strings(rng, 400, 0, 60, alpha) + ["", "é", "ab中", "xyz", "ß" * 20]
    oi, os_, _ = _check(ed, frm, to, metric)
    assert (os_[frm.index("")] == 0.0) and oi[frm.index("")] == 0                # all scores 0: the first index wins


def test_titles_grid_vs_oracle(ed):
    from polyfuzz_b200 import synth
    frm = synth.titles(300, seed=1); to = synth.titles(5000, seed=2)
    for metric in METRICS:
        _check(ed, frm, to, metric)


def test_self_match_duplicates_cutoff_and_big_alphabet(ed):
    rng = np.random.default_rng(3)
    s = _rand_strings(rng, 400, 3, 20, "abcdef") + ["dup", "dup"]
    for metric, cut in (("jaro_winkler", 0.85), ("jaro", 0.8)):
        bi, bs, bd = ed.edit_argbest(s, s, metric, score_cutoff=cut, exclude_self=True)
        oi, os_, od = jaro_oracle.jaro_argbest(s, s, metric, score_cutoff=cut, exclude_self=True, n_threads=NT)
        np.testing.assert_array_equal(bi.cpu().numpy(), oi); np.testing.assert_array_equal(bs.cpu().numpy(), os_)
        np.testing.assert_array_equal(bd.cpu().numpy(), od)
        assert (oi != np.arange(len(s))).all() and (oi == -1).any() and oi[-2] == len(s) - 1 and oi[-1] == len(s) - 2
    # more than 255 distinct code points in the from-list -> alphabet batches
    big = [chr(0x4E00 + i) + chr(0x4E00 + (i * 7) % 600) + "ab" for i in range(600)]
    to = big[::3] + ["ab", "中ab"]
    for metric in METRICS:
        _check(ed, big, to, metric)


def test_to_shards_merge_equals_single_call(ed):
    """Single-GPU emulation of distributed=True: each to-shard staged separately with its global index base and self
    shift, the per-shard bests merged by lev_merge (score desc, global index asc)."""
    import torch
    from polyfuzz_b200.distributed import shard_bounds
    from polyfuzz_b200 import synth
    s = synth.titles(700, seed=4) + ["Alpha", "Alpha"]
    for metric in METRICS:
        whole = ed.edit_argbest(s, s, metric, score_cutoff=0.6, exclude_self=True)
        Q = ed.EditQueries(s)
        parts = []
        for r in range(2):
            lo, hi = shard_bounds(len(s), 2, r)
            T = ed.EditTargets(s[lo:hi])
            parts.append(ed.edit_argbest_staged(Q, T, metric, 0.6, exclude_self=True, self_shift=-lo, to_index_base=lo))
        merged = ed.lev_merge(*(torch.stack([p[c] for p in parts]) for c in range(3)))
        for a, b in zip(whole, merged):
            np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
        oi, os_, od = jaro_oracle.jaro_argbest(s, s, metric, score_cutoff=0.6, exclude_self=True, n_threads=NT)
        np.testing.assert_array_equal(merged[0].cpu().numpy(), oi); np.testing.assert_array_equal(merged[1].cpu().numpy(), os_)
        np.testing.assert_array_equal(merged[2].cpu().numpy(), od)


@pytest.mark.parametrize("normalize", [True, False])
def test_editdistance_frames(normalize):
    from polyfuzz_b200 import EditDistance
    for metric in METRICS:
        name = metric + "_similarity"
        got = EditDistance(n_jobs=1, scorer=name, normalize=normalize).match(FROM, TO)
        oi, os_, _ = jaro_oracle.jaro_argbest(FROM, TO, metric, score_cutoff=float("-inf"))
        assert got.From.tolist() == FROM and got.To.tolist() == [TO[i] for i in oi]
        exp = os_ if not normalize else (os_ - os_.min()) / (os_.max() - os_.min())
        np.testing.assert_array_equal(got.Similarity.to_numpy(), exp)
        # a self-match excludes index i only
        got = EditDistance(scorer=name, normalize=False).match(FROM + ["apple"])
        oi, os_, _ = jaro_oracle.jaro_argbest(FROM + ["apple"], FROM + ["apple"], metric, score_cutoff=float("-inf"), exclude_self=True)
        assert got.To.tolist() == [(FROM + ["apple"])[i] for i in oi] and got.Similarity.tolist() == os_.tolist()


def test_real_movie_titles_sample(ed):
    from polyfuzz_b200 import datasets
    data, kind = datasets.load_movie_titles()
    if kind != "real":
        pytest.skip("the movie-title fixture is not present")
    rng = np.random.default_rng(0)
    rows = np.sort(rng.choice(len(data["Netflix"]), 300, replace=False))
    frm = [data["Netflix"][i] for i in rows]
    _check(ed, frm, data["IMDB"], "jaro_winkler")


def test_rejections(ed):
    with pytest.raises(ValueError, match="distance matrix"):
        ed.edit_argbest(["abc"], ["abd"], "jaro_winkler", want_matrix=True)
    with pytest.raises(ValueError, match="at most"):
        ed.edit_argbest(["x" * 1025], ["y"], "jaro")
    bi, bs, bd = ed.edit_argbest(["x" * 1024], ["x" * 1024, "y"], "jaro")
    assert int(bi[0]) == 0 and float(bs[0]) == 1.0 and int(bd[0]) == 1024


TUTORIAL = """
from polyfuzz import PolyFuzz
from polyfuzz.models import EditDistance
from jellyfish import jaro_winkler_similarity

from_list = ["apple", "apples", "appl", "recal", "house", "similarity"]
to_list = ["apple", "apples", "mouse"]

jellyfish_matcher = EditDistance(n_jobs=1, scorer=jaro_winkler_similarity)
model = PolyFuzz(jellyfish_matcher).match(from_list, to_list)
"""


def test_tutorial_snippet_through_reference_orchestrator(monkeypatch):
    """The reference tutorial's jellyfish example (docs/tutorial/models/models.md:49-59), verbatim: first with the
    reference's own EditDistance calling a stand-in jellyfish (the CPU oracle), then after polyfuzz_b200.install(), which
    puts this package's EditDistance behind the same names.  Both frames must be equal."""
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference orchestrator) was not built")
    import types
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    from oracle import ref_shim
    ref_shim.REFERENCE_ROOT = REF
    ref_shim.install()
    jf = types.ModuleType("jellyfish")

    def jaro_winkler_similarity(s1, s2):
        return jaro_oracle.jaro_winkler_similarity(s1, s2)

    def jaro_similarity(s1, s2):
        return jaro_oracle.jaro_similarity(s1, s2)

    jf.jaro_winkler_similarity, jf.jaro_similarity = jaro_winkler_similarity, jaro_similarity
    monkeypatch.setitem(sys.modules, "jellyfish", jf)
    import polyfuzz.models as pm
    import polyfuzz.polyfuzz as pp
    for mod in (pm, pp):                                   # install() rebinds these; undone after the test
        for name in ("TFIDF", "RapidFuzz", "EditDistance", "Embeddings"):
            if hasattr(mod, name):
                monkeypatch.setattr(mod, name, getattr(mod, name))
    ns_ref = {}
    exec(TUTORIAL, ns_ref)
    ref = ns_ref["model"].get_matches()
    import polyfuzz_b200
    polyfuzz_b200.install()
    ns_gpu = {}
    exec(TUTORIAL, ns_gpu)
    assert isinstance(ns_gpu["jellyfish_matcher"], polyfuzz_b200.EditDistance)
    got = ns_gpu["model"].get_matches()
    assert list(got.columns) == list(ref.columns) == ["From", "To", "Similarity"]
    assert got.From.tolist() == ref.From.tolist() and got.To.tolist() == ref.To.tolist()
    np.testing.assert_array_equal(got.Similarity.to_numpy(dtype=np.float64), ref.Similarity.to_numpy(dtype=np.float64))
