"""GPU parity tests of K3's sequence metrics (csrc/pfz_lev.cu: NORM_INDEL / NORM_LCSSEQ on lev_kernel's LCS recurrence, NORM_HAMMING /
NORM_PREFIX / NORM_POSTFIX in pos_kernel) against the plain-Python oracle (tests/seq_oracle.py).  Indices, scores and distances
are compared with ==: the kernel's score is the oracle's IEEE expression 1 - d/M on the same integers."""
import math
import os

import numpy as np
import pytest
import torch

import seq_oracle
from seq_oracle import METRICS

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
REF = os.path.join(ROOT, "oracle", "_ref")
EDGES = [0, 1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024]
NAME = {"norm_indel": "indel", "norm_lcsseq": "lcsseq", "norm_hamming": "hamming", "norm_prefix": "prefix", "norm_postfix": "postfix"}


@pytest.fixture(scope="module")
def ed():
    from polyfuzz_b200 import editdist
    return editdist


class Grid:
    """The oracle's (D, S) of every metric over from x to, the LCS matrix computed once."""

    def __init__(self, frm, to):
        self.frm, self.to = frm, to
        lcs = seq_oracle.lcs_matrix(frm, to)
        self.D, self.S = {}, {}
        for metric in METRICS:
            self.D[metric], _, self.S[metric] = seq_oracle.matrices(metric, frm, to, lcs)

    def topk(self, metric, k, cutoff=0.0, exclude_self=False, self_shift=0, allowed=None):
        return seq_oracle.topk_from(self.S[metric], self.D[metric], k, cutoff, exclude_self, self_shift, allowed)


def _check_argbest(got, grid, metric, cutoff=0.0, exclude_self=False):
    oi, os_, od = (a[:, 0] for a in grid.topk(metric, 1, cutoff, exclude_self))
    np.testing.assert_array_equal(got[0].cpu().numpy(), oi, err_msg=metric)
    np.testing.assert_array_equal(got[1].cpu().numpy(), os_, err_msg=metric)
    np.testing.assert_array_equal(got[2].cpu().numpy(), od, err_msg=metric)
    return oi


def _check_topk(got, grid, metric, k, cutoff=0.0, exclude_self=False):
    oi, os_, _ = grid.topk(metric, k, cutoff, exclude_self)
    np.testing.assert_array_equal(got[0].cpu().numpy(), oi, err_msg=f"{metric} k={k}")
    np.testing.assert_array_equal(got[1].cpu().numpy(), os_, err_msg=f"{metric} k={k}")


def _rand(rng, n, alpha):
    return "".join(alpha[i] for i in rng.integers(0, len(alpha), n))


def _edge_lists(seed, alpha="abcdeé中😀"):
    """From-strings at every word-class edge (0 .. 1 024 code points) plus short ones.  To-strings: short random ones, and for
    every edge string its prefixes and suffixes with new ends, one substitution, shorter and longer copies (unequal lengths on
    both sides), plus three of 2 000+ code points."""
    rng = np.random.default_rng(seed)
    frm = [_rand(rng, L, alpha) for L in EDGES] + [_rand(rng, int(rng.integers(0, 41)), alpha) for _ in range(30)]
    to = [_rand(rng, int(rng.integers(0, 81)), alpha) for _ in range(150)]
    for s in frm[:len(EDGES)]:
        if not s:
            continue
        cut = int(rng.integers(0, len(s) + 1))
        to += [s[:cut] + _rand(rng, int(rng.integers(0, 6)), alpha), _rand(rng, int(rng.integers(0, 6)), alpha) + s[cut:]]
        p = int(rng.integers(0, len(s)))
        to += [s[:p] + ("x" if s[p] != "x" else "y") + s[p + 1:], s[:-1], s + _rand(rng, 3, alpha)]
    long_ = [frm[-31] * 2 + "ab", _rand(rng, 2050, alpha), _rand(rng, 1500, alpha) + frm[-31]]
    to += long_ + ["", frm[20], frm[-31]]
    assert max(map(len, to)) >= 2000 and max(map(len, frm)) == 1024
    return frm, to


@pytest.fixture(scope="module")
def edges():
    frm, to = _edge_lists(7)
    return Grid(frm, to)


@pytest.mark.parametrize("metric", METRICS)
def test_word_class_edges_argbest_and_topk(ed, edges, metric):
    Q, T = ed.EditQueries(edges.frm), ed.EditTargets(edges.to)
    for n_splits in (1, 3, None):
        _check_argbest(ed.edit_argbest_staged(Q, T, metric, 0.0, n_splits=n_splits), edges, metric)
        for k in (1, 3, 32):
            _check_topk(ed.edit_topk_staged(Q, T, k, metric, 0.0, n_splits=n_splits), edges, metric, k)
    bi, bs, _ = ed.edit_argbest_staged(Q, T, metric, float("-inf"))
    ti, tv = ed.edit_topk_staged(Q, T, 10, metric, float("-inf"))
    np.testing.assert_array_equal(ti[:, 0].cpu().numpy(), bi.cpu().numpy())
    np.testing.assert_array_equal(tv[:, 0].cpu().numpy(), bs.cpu().numpy())


@pytest.fixture(scope="module")
def unequal():
    rng = np.random.default_rng(11)
    frm = [_rand(rng, L, "ab") for L in range(10) for _ in range(3)]
    to = [_rand(rng, L, "ab") for L in range(10) for _ in range(4)] + [f + "b" for f in frm[::2]] + ["a" + f for f in frm[1::2]]
    return Grid(frm, to)


@pytest.mark.parametrize("metric", METRICS)
def test_unequal_lengths_both_sides(ed, unequal, metric):
    """Every pair of lengths 0..9 over a two-letter alphabet, from-side and to-side: prefixes, suffixes and the Hamming surplus
    at every offset of the 4-symbol words."""
    grid = unequal
    frm, to = grid.frm, grid.to
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    _check_argbest(ed.edit_argbest_staged(Q, T, metric, float("-inf")), grid, metric, float("-inf"))
    _check_topk(ed.edit_topk_staged(Q, T, 32, metric, float("-inf")), grid, metric, 32, float("-inf"))


@pytest.fixture(scope="module")
def batches():
    big = [chr(0x4E00 + i) + chr(0x4E00 + (i * 7) % 600) + "abc" for i in range(600)]
    out = ["Ж", "Я", "ю"]
    assert not set("".join(out)) & set("".join(big))
    to = big[::3] + ["ab", "中ab"] + [s[1] + "x" + s[0] + s[2:] for s in big[1::7]]
    to += [o + s[1:] for s in big[:40:5] for o in out] + [s[:2] + o + s[3:] for s in big[:40:5] for o in out]
    to += [s[:-1] + o for s in big[:40:5] for o in out] + [s + o for s in big[:40:5] for o in out]
    assert len(set("".join(big))) > 255
    return Grid(big, to)


@pytest.mark.parametrize("metric", METRICS)
def test_alphabet_batches_and_text_only_symbols(ed, batches, metric):
    """A from-list of 600+ distinct code points (several alphabet batches); to-strings that differ from each other only in code
    points no from-string has (symbol 0, which equals no pattern symbol), at the start, the middle and the end."""
    grid = batches
    big, to = grid.frm, grid.to
    _check_argbest(ed.edit_argbest(big, to, metric, 0.0), grid, metric)
    _check_topk(ed.edit_topk(big, to, 5, metric, 0.0), grid, metric, 5)


@pytest.fixture(scope="module")
def selfs():
    rng = np.random.default_rng(3)
    s = [_rand(rng, int(rng.integers(3, 21)), "abcdef") for _ in range(300)] + ["dup", "dup", "dpu", "", ""]
    return Grid(s, s)


@pytest.mark.parametrize("metric", METRICS)
def test_self_match_and_cutoffs_at_achievable_scores(ed, selfs, metric):
    """Cutoffs equal to scores the list achieves (the pair is kept) and the next double up (it is rejected)."""
    grid = selfs
    s = grid.frm
    S = grid.S[metric].copy()
    np.fill_diagonal(S, -1.0)
    vals = np.unique(S[S >= 0])
    cuts = {float(vals[len(vals) // 2]), float(vals[-2]), float(S.max(axis=1)[7]), float(vals[-1])}
    cuts |= {math.nextafter(c, math.inf) for c in list(cuts)} | {0.0}
    Q = ed.EditQueries(s); T = ed.EditTargets(s)
    for c in sorted(cuts):
        oi = _check_argbest(ed.edit_argbest_staged(Q, T, metric, c, exclude_self=True), grid, metric, c, True)
        assert (oi != np.arange(len(s))).all()
        for k in (3, 32):
            _check_topk(ed.edit_topk_staged(Q, T, k, metric, c, exclude_self=True), grid, metric, k, c, True)
    kept = float(S.max(axis=1)[7])
    got = ed.edit_argbest_staged(Q, T, metric, kept, exclude_self=True)
    assert float(got[1][7]) == kept
    got = ed.edit_argbest_staged(Q, T, metric, math.nextafter(kept, math.inf), exclude_self=True)
    assert int(got[0][7]) == -1


@pytest.mark.parametrize("metric", METRICS)
def test_candidate_mode_equals_all_pairs_on_each_list(ed, edges, metric):
    rng = np.random.default_rng(9)
    frm, to = edges.frm, edges.to
    c = 40
    cand = np.full((len(frm), c), -1, dtype=np.int32)
    for i in range(len(frm)):
        n_c = int(rng.integers(0, c + 1))
        cand[i, rng.permutation(c)[:n_c]] = rng.permutation(len(to))[:n_c]        # shuffled, with -1 slots anywhere
    cand[3] = -1
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    d_cand = torch.from_numpy(cand).cuda()
    for k in (1, 3, 32):
        for cutoff, excl in ((0.0, False), (0.4, True)):
            got = ed.edit_cand_topk_staged(Q, T, d_cand, k, metric, cutoff, exclude_self=excl)
            ei, ev, edist = edges.topk(metric, k, cutoff, excl, allowed=cand)
            np.testing.assert_array_equal(got[0].cpu().numpy().reshape(len(frm), -1), ei)
            np.testing.assert_array_equal(got[1].cpu().numpy().reshape(len(frm), -1), ev)
            if k == 1:
                np.testing.assert_array_equal(got[2].cpu().numpy(), edist[:, 0])


@pytest.fixture(scope="module")
def titles():
    from polyfuzz_b200 import synth
    s = synth.titles(500, seed=4) + ["Alpha", "Alpha", "lApha", "Alphas", "The Alpha"]
    return Grid(s, s)


@pytest.mark.parametrize("metric", METRICS)
def test_to_shards_merge_equals_single_call(ed, titles, metric):
    """Single-GPU emulation of distributed=True: each to-shard staged separately with its global index base and self shift;
    arg-best merged by lev_merge, top-k by merge_topk_any (pfz_topk_merge)."""
    from polyfuzz_b200.distributed import merge_topk_any, shard_bounds
    grid = titles
    s = grid.frm
    whole = ed.edit_argbest(s, s, metric, 0.5, exclude_self=True)
    wtop = ed.edit_topk(s, s, 5, metric, 0.5, exclude_self=True)
    Q = ed.EditQueries(s)
    parts, tparts = [], []
    for r in range(2):
        lo, hi = shard_bounds(len(s), 2, r)
        T = ed.EditTargets(s[lo:hi])
        parts.append(ed.edit_argbest_staged(Q, T, metric, 0.5, exclude_self=True, self_shift=-lo, to_index_base=lo))
        tparts.append(ed.edit_topk_staged(Q, T, 5, metric, 0.5, exclude_self=True, self_shift=-lo, to_index_base=lo))
    merged = ed.lev_merge(*(torch.stack([p[c] for p in parts]) for c in range(3)))
    for a, b in zip(whole, merged):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    _check_argbest(merged, grid, metric, 0.5, True)
    mi, mv = merge_topk_any(torch.stack([t[0] for t in tparts]), torch.stack([t[1] for t in tparts]), 5)
    for a, b in zip(wtop, (mi, mv)):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    _check_topk((mi, mv), grid, metric, 5, 0.5, True)


@pytest.mark.parametrize("metric", METRICS)
def test_matcher_frames(metric):
    """EditDistance (normalize, top_n, candidates) and RapidFuzz (score_cutoff on 0..1, top_n) frames against the oracle."""
    from polyfuzz_b200 import EditDistance, RapidFuzz, TFIDF
    frm = ["kitten", "Jhon Smtih", "Micorsoft", "apple", "appel", "house", "Intl Business Machines", "SKU-0042-B", "SW1A 1AA"]
    to = ["sitting", "XY", "Joan Smyth", "John Smith", "Microsoft", "apple", "apples", "mouse", "International Business Machines",
          "SKU-0042-A", "SKU-0043-B", "SW1A 2AA", "NW1A 1AA", "appl"]
    grid = Grid(frm, to)
    name = NAME[metric]
    df = EditDistance(scorer=name, normalize=False).match(frm, to)
    oi, os_, _ = (a[:, 0] for a in grid.topk(metric, 1, float("-inf")))
    assert df.To.tolist() == [to[i] for i in oi] and df.Similarity.tolist() == os_.tolist()
    df = EditDistance(scorer=name, normalize=True).match(frm, to)
    np.testing.assert_array_equal(df.Similarity.to_numpy(), (os_ - os_.min()) / (os_.max() - os_.min()))
    df = EditDistance(scorer=name, normalize=False, top_n=3).match(frm, to)
    ti, tv, _ = grid.topk(metric, 3, float("-inf"))
    assert df.To_3.tolist() == [to[j] for j in ti[:, 2]] and df.Similarity_3.tolist() == tv[:, 2].tolist()
    df = RapidFuzz(scorer=name, score_cutoff=0.6).match(frm, to)
    oi, os_, _ = (a[:, 0] for a in grid.topk(metric, 1, 0.6))
    assert df.To.tolist() == [to[i] if i >= 0 else None for i in oi]
    assert df.Similarity.tolist() == [s if i >= 0 else 0.0 for s, i in zip(os_, oi)]
    df = RapidFuzz(scorer=name, score_cutoff=0.4, top_n=2).match(frm, to)
    ti, tv, _ = grid.topk(metric, 2, 0.4)
    assert df.To_2.tolist() == [to[j] if j >= 0 else None for j in ti[:, 1]]
    assert df.Similarity_2.tolist() == [v if j >= 0 else 0.0 for v, j in zip(tv[:, 1], ti[:, 1])]
    tf = TFIDF(n_gram_range=(3, 3), min_similarity=0.0, top_n=4)
    cand = tf.match_arrays(frm, to)[0].cpu().numpy()
    df = RapidFuzz(scorer=name, top_n=2, candidates=tf).match(frm, to)
    ci, cv, _ = grid.topk(metric, 2, 0.0, allowed=cand)
    assert df.To.tolist() == [to[j] if j >= 0 else None for j in ci[:, 0]]
    assert df.Similarity_2.tolist() == [v if j >= 0 else 0.0 for v, j in zip(cv[:, 1], ci[:, 1])]


def test_kept_to_side_across_re_train_false(monkeypatch, edges):
    from polyfuzz_b200 import EditDistance, RapidFuzz, editdist
    made = []
    real = editdist.EditTargets
    monkeypatch.setattr(editdist, "EditTargets", lambda lst: made.append(len(lst)) or real(lst))
    frm, to = edges.frm, edges.to
    for m, metric in ((EditDistance(scorer="lcsseq", normalize=False), "norm_lcsseq"), (RapidFuzz(scorer="postfix", top_n=3),
                                                                                        "norm_postfix")):
        made.clear()
        first = m.match(frm, to)
        again = m.match(frm, list(to), re_train=False)
        assert made == [len(to)] and first.equals(again)
        m.match(frm[:5], to, re_train=False)
        assert made == [len(to)]
    oi, _, _ = edges.topk("norm_postfix", 3, 0.0)
    assert again.To_3.tolist() == [to[j] if j >= 0 else None for j in oi[:, 2]]


def test_real_movie_titles_sample(ed):
    from polyfuzz_b200 import datasets
    data, kind = datasets.load_movie_titles()
    if kind != "real":
        pytest.skip("the movie-title fixture is not present")
    rng = np.random.default_rng(0)
    rows = np.sort(rng.choice(len(data["Netflix"]), 8, replace=False))
    frm, to = [data["Netflix"][i] for i in rows], data["IMDB"]
    grid = Grid(frm, to)
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    for metric in METRICS:
        _check_argbest(ed.edit_argbest_staged(Q, T, metric, 0.0), grid, metric)
        _check_topk(ed.edit_topk_staged(Q, T, 10, metric, 0.0), grid, metric, 10)


SNIPPET = """
from polyfuzz import PolyFuzz
from polyfuzz.models import EditDistance

from_list = ["kitten", "Jhon Smtih", "Micorsoft", "apple", "appel", "house", "Intl Business Machines"]
to_list = ["sitting", "XY", "Joan Smyth", "John Smith", "Microsoft", "apple", "apples", "mouse", "International Business Machines"]

model = PolyFuzz(EditDistance(n_jobs=1, scorer=SCORER)).fit(from_list, to_list)
matches = model.get_matches()
new = model.transform(["Mikrosoft", "Jon Smith", "apel", "Intl Bus. Machines"])["EditDistance"]
"""


def test_reference_orchestrator(monkeypatch):
    """PolyFuzz(EditDistance(scorer="lcsseq")).fit / .transform through the unmodified reference orchestrator: first with the
    reference's own EditDistance calling a stand-in LCSseq scorer (the oracle, named lcs_seq), then after polyfuzz_b200.install()
    with the stand-in and with the name "lcsseq".  The frames must be equal."""
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference orchestrator) was not built")
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    from oracle import ref_shim
    ref_shim.REFERENCE_ROOT = REF
    ref_shim.install()

    def lcs_seq(s1, s2):
        return seq_oracle.similarity("norm_lcsseq", s1, s2)

    import polyfuzz.models as pm
    import polyfuzz.polyfuzz as pp
    for mod in (pm, pp):                                   # install() rebinds these; undone after the test
        for name in ("TFIDF", "RapidFuzz", "EditDistance", "Embeddings"):
            if hasattr(mod, name):
                monkeypatch.setattr(mod, name, getattr(mod, name))
    ns_ref = {"SCORER": lcs_seq}
    exec(SNIPPET, ns_ref)
    import polyfuzz_b200
    polyfuzz_b200.install()
    for scorer in (lcs_seq, "lcsseq"):
        ns_gpu = {"SCORER": scorer}
        exec(SNIPPET, ns_gpu)
        for key in ("matches", "new"):
            got, ref = ns_gpu[key], ns_ref[key]
            assert list(got.columns) == list(ref.columns)
            assert got.From.tolist() == ref.From.tolist() and got.To.tolist() == ref.To.tolist()
            np.testing.assert_array_equal(got.Similarity.to_numpy(dtype=np.float64), ref.Similarity.to_numpy(dtype=np.float64))
    assert ns_gpu["matches"].To.tolist()[-1] == "International Business Machines"
