"""GPU parity tests of weighted Levenshtein in K3 (csrc/pfz_lev.cu, wlev_kernel: the Indel form, and the unit-Levenshtein bounds
with a queued exact DP) against the int64 Wagner-Fischer of the CPU oracle (tests/wlev_oracle.c).  Indices, scores and distances
are compared with ==: the kernel's score is the oracle's IEEE expression 1 - D/M on the same integers."""
import functools
import os

import numpy as np
import pytest
import torch

import wlev_oracle

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
REF = os.path.join(ROOT, "oracle", "_ref")
NT = os.cpu_count() or 1
I32_MAX = 2**31 - 1
GRID = [(0, 0, 0), (0, 1, 1), (1, 0, 3), (1, 1, 0), (1, 3, 2), (5, 2, 7), (1, 1, 2), (3, 3, 9), (2, 2, 2), (65535, 1, 65535)]
KS = [1, 3, 32]
EDGES = [0, 1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024]


@pytest.fixture(scope="module")
def ed():
    from polyfuzz_b200 import editdist
    return editdist


def _rand_strings(rng, n, lo, hi, alpha):
    return ["".join(alpha[i] for i in rng.integers(0, len(alpha), rng.integers(lo, hi + 1))) for _ in range(n)]


def _mutate(rng, s, n_edits, alpha):
    """s with n_edits random substitutions, insertions and deletions: a near match whose bounds rarely meet."""
    s = list(s)
    for _ in range(n_edits):
        op, p = rng.integers(0, 3), int(rng.integers(0, len(s) + 1))
        c = alpha[int(rng.integers(0, len(alpha)))]
        if op == 0 and p < len(s):
            s[p] = c
        elif op == 1:
            s.insert(p, c)
        elif p < len(s):
            del s[p]
    return "".join(s)


def _check_argbest(ed, got, frm, to, weights, cutoff=0.0, exclude_self=False):
    oi, os_, od = wlev_oracle.wlev_argbest(frm, to, weights, cutoff, exclude_self, n_threads=NT)
    np.testing.assert_array_equal(got[0].cpu().numpy(), oi)
    np.testing.assert_array_equal(got[1].cpu().numpy(), os_)
    np.testing.assert_array_equal(got[2].cpu().numpy(), np.minimum(od, I32_MAX))
    return oi, os_


def _check_topk(got, frm, to, weights, k, cutoff=0.0, exclude_self=False):
    oi, os_, _ = wlev_oracle.wlev_topk(frm, to, weights, k, cutoff, exclude_self, n_threads=NT)
    np.testing.assert_array_equal(got[0].cpu().numpy(), oi)
    np.testing.assert_array_equal(got[1].cpu().numpy(), os_)


def _edge_lists(seed, alpha="abcdeé中"):
    """From-strings at every word-class edge (0 .. 1 024 code points) plus short ones; to-strings: short random ones, near
    matches of every from-string, and three of 2 000+ code points."""
    rng = np.random.default_rng(seed)
    frm = ["".join(alpha[i] for i in rng.integers(0, len(alpha), L)) for L in EDGES] + _rand_strings(rng, 30, 0, 40, alpha)
    near = [_mutate(rng, s, int(rng.integers(1, 6)), alpha) for s in frm[:len(EDGES)] for _ in range(2)]
    long = [_mutate(rng, frm[-31] * 2, 40, alpha), "".join(alpha[i] for i in rng.integers(0, len(alpha), 2050)), frm[-31][:600] * 4]
    to = _rand_strings(rng, 200, 0, 80, alpha) + near + long + ["", frm[20], frm[-31]]
    assert max(map(len, to)) >= 2000 and max(map(len, frm)) == 1024
    return frm, to


@pytest.mark.parametrize("weights", GRID)
def test_word_class_edges_argbest_and_topk(ed, weights):
    frm, to = _edge_lists(sum(weights) % 101)
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    for n_splits in (1, 3, None):
        _check_argbest(ed, ed.edit_wlev_argbest_staged(Q, T, weights, 0.0, n_splits=n_splits), frm, to, weights)
    for k in KS:
        for n_splits in (1, 3, None):
            _check_topk(ed.edit_wlev_topk_staged(Q, T, k, weights, 0.0, n_splits=n_splits), frm, to, weights, k)
    bi, bs, _ = ed.edit_wlev_argbest_staged(Q, T, weights, float("-inf"))
    ti, tv = ed.edit_wlev_topk_staged(Q, T, 10, weights, float("-inf"))
    np.testing.assert_array_equal(ti[:, 0].cpu().numpy(), bi.cpu().numpy())
    np.testing.assert_array_equal(tv[:, 0].cpu().numpy(), bs.cpu().numpy())


@pytest.mark.parametrize("weights", [(65535, 1, 65535), (1, 65535, 65535), (65535, 65535, 1), (32767, 32767, 65535)])
def test_long_to_strings_past_int32_at_the_weight_cap(ed, weights):
    """To-strings of 40 000 code points: at the weight cap D and M pass 2^31 (65 535 per insertion), which int32 state would
    wrap; with costly deletions the DP state spans [-m wi, m wd].  Scores stay exact; the arg-best distance saturates at
    2^31 - 1."""
    rng = np.random.default_rng(5)
    alpha = "abcdé"
    frm = ["".join(alpha[i] for i in rng.integers(0, len(alpha), L)) for L in (1024, 700, 64, 5, 0)]
    to = [(frm[0] + "x") * 39, _mutate(rng, frm[1] * 57, 300, alpha), "".join(alpha[i] for i in rng.integers(0, len(alpha), 40000)),
          frm[2] * 5, frm[3], ""]
    D, M = wlev_oracle.wlev_matrix(frm, to, weights, n_threads=NT)
    if weights[0] == 65535:                                 # costly insertions: 40 000 of them pass 2^31
        assert M.max() > I32_MAX and D.max() > I32_MAX
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    for cutoff in (float("-inf"), 0.0):
        _check_argbest(ed, ed.edit_wlev_argbest_staged(Q, T, weights, cutoff), frm, to, weights, cutoff)
        _check_topk(ed.edit_wlev_topk_staged(Q, T, 6, weights, cutoff), frm, to, weights, 6, cutoff)


@pytest.mark.parametrize("weights", [(5, 2, 7), (1, 1, 2), (0, 1, 1)])
def test_alphabet_batches(ed, weights):
    big = [chr(0x4E00 + i) + chr(0x4E00 + (i * 7) % 600) + "abc" for i in range(600)]
    to = big[::3] + ["ab", "中ab"] + [s[1] + "x" + s[0] + s[2:] for s in big[1::7]]
    assert len(set("".join(big))) > 255
    _check_argbest(ed, ed.edit_wlev_argbest(big, to, weights), big, to, weights)
    _check_topk(ed.edit_wlev_topk(big, to, 5, weights), big, to, weights, 5)


@pytest.mark.parametrize("weights", [(1, 3, 2), (5, 2, 7), (1, 1, 2), (1, 1, 0)])
def test_self_match_and_cutoffs_at_achievable_scores(ed, weights):
    """Cutoffs equal to scores the list achieves (and the doubles next to them): a pair whose score equals the cutoff is kept."""
    import math
    rng = np.random.default_rng(3)
    s = _rand_strings(rng, 300, 3, 20, "abcdef") + ["dup", "dup", "dpu", "", ""]
    S = wlev_oracle.score_matrix(s, s, weights, n_threads=NT)
    np.fill_diagonal(S, -1.0)
    vals = np.unique(S[S >= 0])
    cuts = {float(vals[len(vals) // 2]), float(vals[-2]), float(S.max(axis=1)[7]), float(vals[-1])}
    cuts |= {math.nextafter(c, math.inf) for c in list(cuts)} | {0.0}
    Q = ed.EditQueries(s); T = ed.EditTargets(s)
    for c in sorted(cuts):
        oi, _ = _check_argbest(ed, ed.edit_wlev_argbest_staged(Q, T, weights, c, exclude_self=True), s, s, weights, c, True)
        assert (oi != np.arange(len(s))).all()
        for k in (3, 32):
            _check_topk(ed.edit_wlev_topk_staged(Q, T, k, weights, c, exclude_self=True), s, s, weights, k, c, True)


@pytest.mark.parametrize("w", [1, 2, 65535])
def test_uniform_weights_equal_norm_lev_and_the_generic_path(ed, w):
    """(w, w, w): the matcher's frames equal scorer="levenshtein"'s; the host routes them to norm_lev, and pfz_wlev_rows itself
    (bounds that always meet) gives the same rows."""
    from polyfuzz_b200 import EditDistance, RapidFuzz
    frm, to = _edge_lists(11)
    p = functools.partial(wlev_oracle.normalized_similarity, weights=(w, w, w))
    for cls, kw in ((EditDistance, {}), (EditDistance, {"top_n": 4}), (RapidFuzz, {"score_cutoff": 0.3}),
                    (RapidFuzz, {"score_cutoff": 0.2, "top_n": 3})):
        got = cls(scorer=p, **kw).match(frm, to)
        ref = cls(scorer="levenshtein", **kw).match(frm, to)
        assert got.equals(ref)
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    ref = ed.edit_argbest_staged(Q, T, "norm_lev", 0.0)
    gen = ed._edit_rows(Q, T, None, 0.0, False, 0, 0, weights=(w, w, w))
    for a, b in zip(ref[:2], gen[:2]):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    np.testing.assert_array_equal(np.minimum(ref[2].cpu().numpy().astype(np.int64) * w, I32_MAX), gen[2].cpu().numpy())
    ti, tv = ed.edit_topk_staged(Q, T, 7, "norm_lev", 0.0)
    gi, gv = ed._edit_rows(Q, T, None, 0.0, False, 0, 7, weights=(w, w, w))
    np.testing.assert_array_equal(ti.cpu().numpy(), gi.cpu().numpy()); np.testing.assert_array_equal(tv.cpu().numpy(), gv.cpu().numpy())


@pytest.mark.parametrize("weights", [(1, 1, 2), (3, 3, 9), (2, 2, 5)])
def test_indel_form_equals_the_generic_dp(ed, weights):
    """(w, w, >= 2w) runs the LCS recurrence; its frames equal the oracle's full weighted DP."""
    from polyfuzz_b200 import EditDistance
    frm, to = _edge_lists(23)
    p = functools.partial(wlev_oracle.normalized_similarity, weights=weights)
    got = EditDistance(scorer=p, normalize=False).match(frm, to)
    oi, os_, _ = wlev_oracle.wlev_argbest(frm, to, weights, float("-inf"), n_threads=NT)
    assert got.To.tolist() == [to[i] for i in oi] and got.Similarity.tolist() == os_.tolist()
    got = EditDistance(scorer=p, normalize=False, top_n=5).match(frm, to)
    ti, tv, _ = wlev_oracle.wlev_topk(frm, to, weights, 5, float("-inf"), n_threads=NT)
    assert got.To_5.tolist() == [to[j] for j in ti[:, 4]] and got.Similarity_5.tolist() == tv[:, 4].tolist()


@pytest.mark.parametrize("weights", [(5, 2, 7), (1, 1, 2), (1, 0, 3)])
def test_candidate_mode_equals_all_pairs_on_each_list(ed, weights):
    rng = np.random.default_rng(9)
    frm, to = _edge_lists(31)
    c = 40
    cand = np.full((len(frm), c), -1, dtype=np.int32)
    for i in range(len(frm)):
        n_c = int(rng.integers(0, c + 1))
        cand[i, rng.permutation(c)[:n_c]] = rng.permutation(len(to))[:n_c]        # shuffled, with -1 slots anywhere
    if len(frm) > 3:
        cand[3] = -1
    Q, T = ed.EditQueries(frm), ed.EditTargets(to)
    d_cand = torch.from_numpy(cand).cuda()
    S = wlev_oracle.score_matrix(frm, to, weights, n_threads=NT)
    D, _ = wlev_oracle.wlev_matrix(frm, to, weights, n_threads=NT)
    for k in (1, 3, 32):
        for cutoff, excl in ((0.0, False), (0.4, True)):
            got = ed.edit_wlev_cand_topk_staged(Q, T, d_cand, k, weights, cutoff, exclude_self=excl)
            for i in range(len(frm)):
                js = np.array([j for j in cand[i] if j >= 0 and S[i, j] >= cutoff and not (excl and j == i)], dtype=np.int64)
                js = js[np.lexsort((js, -S[i, js]))][:k] if len(js) else js
                ei = np.full(k, -1, np.int32); ev = np.zeros(k); ei[:len(js)] = js; ev[:len(js)] = S[i, js]
                gi = got[0][i].cpu().numpy().reshape(-1); gv = got[1][i].cpu().numpy().reshape(-1)
                np.testing.assert_array_equal(gi, ei[:len(gi)]); np.testing.assert_array_equal(gv, ev[:len(gv)])
                if k == 1:
                    assert int(got[2][i]) == (min(int(D[i, js[0]]), I32_MAX) if len(js) else -1)


@pytest.mark.parametrize("weights", [(5, 2, 7), (1, 1, 2)])
def test_to_shards_merge_equals_single_call(ed, weights):
    """Single-GPU emulation of distributed=True: each to-shard staged separately with its global index base and self shift;
    arg-best merged by lev_merge, top-k by merge_topk_any (pfz_topk_merge)."""
    from polyfuzz_b200 import synth
    from polyfuzz_b200.distributed import merge_topk_any, shard_bounds
    s = synth.titles(700, seed=4) + ["Alpha", "Alpha", "lApha", "lpAha"]
    whole = ed.edit_wlev_argbest(s, s, weights, 0.5, exclude_self=True)
    wtop = ed.edit_wlev_topk(s, s, 5, weights, 0.5, exclude_self=True)
    Q = ed.EditQueries(s)
    parts, tparts = [], []
    for r in range(2):
        lo, hi = shard_bounds(len(s), 2, r)
        T = ed.EditTargets(s[lo:hi])
        parts.append(ed.edit_wlev_argbest_staged(Q, T, weights, 0.5, exclude_self=True, self_shift=-lo, to_index_base=lo))
        tparts.append(ed.edit_wlev_topk_staged(Q, T, 5, weights, 0.5, exclude_self=True, self_shift=-lo, to_index_base=lo))
    merged = ed.lev_merge(*(torch.stack([p[c] for p in parts]) for c in range(3)))
    for a, b in zip(whole, merged):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    _check_argbest(ed, merged, s, s, weights, 0.5, True)
    mi, mv = merge_topk_any(torch.stack([t[0] for t in tparts]), torch.stack([t[1] for t in tparts]), 5)
    for a, b in zip(wtop, (mi, mv)):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    _check_topk((mi, mv), s, s, weights, 5, 0.5, True)


def test_kept_to_side_across_re_train_false(monkeypatch):
    from polyfuzz_b200 import EditDistance, RapidFuzz, editdist
    made = []
    real = editdist.EditTargets
    monkeypatch.setattr(editdist, "EditTargets", lambda lst: made.append(len(lst)) or real(lst))
    frm, to = _edge_lists(41)
    p = functools.partial(wlev_oracle.normalized_similarity, weights=(5, 2, 7))
    for m in (EditDistance(scorer=p, normalize=False), RapidFuzz(scorer=p, top_n=3)):
        made.clear()
        first = m.match(frm, to)
        again = m.match(frm, list(to), re_train=False)
        assert made == [len(to)] and first.equals(again)
        m.match(frm[:5], to, re_train=False)
        assert made == [len(to)]
    oi, os_, _ = wlev_oracle.wlev_topk(frm, to, (5, 2, 7), 3, 0.0, n_threads=NT)
    assert again.To_3.tolist() == [to[j] if j >= 0 else None for j in oi[:, 2]]


SNIPPET = """
from polyfuzz import PolyFuzz
from polyfuzz.models import EditDistance

from_list = ["kitten", "Jhon Smtih", "Micorsoft", "apple", "appel", "house", "similarity"]
to_list = ["sitting", "XY", "Joan Smyth", "John Smith", "Microsoft", "apple", "apples", "mouse"]

model = PolyFuzz(EditDistance(n_jobs=1, scorer=SCORER)).fit(from_list, to_list)
matches = model.get_matches()
new = model.transform(["Mikrosoft", "Jon Smith", "apel"])["EditDistance"]
"""


@pytest.mark.parametrize("weights", [(5, 2, 7), (1, 1, 2)])
def test_reference_orchestrator(monkeypatch, weights):
    """PolyFuzz(EditDistance(scorer=partial(...))).fit / .transform through the unmodified reference orchestrator: first with the
    reference's own EditDistance calling the partial of a stand-in (the CPU oracle, named like rapidfuzz's), then after
    polyfuzz_b200.install().  The frames must be equal."""
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference orchestrator) was not built")
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    from oracle import ref_shim
    ref_shim.REFERENCE_ROOT = REF
    ref_shim.install()
    import polyfuzz.models as pm
    import polyfuzz.polyfuzz as pp
    for mod in (pm, pp):                                   # install() rebinds these; undone after the test
        for name in ("TFIDF", "RapidFuzz", "EditDistance", "Embeddings"):
            if hasattr(mod, name):
                monkeypatch.setattr(mod, name, getattr(mod, name))
    scorer = functools.partial(wlev_oracle.normalized_similarity, weights=weights)
    ns_ref = {"SCORER": scorer}
    exec(SNIPPET, ns_ref)
    import polyfuzz_b200
    polyfuzz_b200.install()
    ns_gpu = {"SCORER": scorer}
    exec(SNIPPET, ns_gpu)
    for key in ("matches", "new"):
        got, ref = ns_gpu[key], ns_ref[key]
        assert list(got.columns) == list(ref.columns)
        assert got.From.tolist() == ref.From.tolist() and got.To.tolist() == ref.To.tolist()
        np.testing.assert_array_equal(got.Similarity.to_numpy(dtype=np.float64), ref.Similarity.to_numpy(dtype=np.float64))
    assert ns_gpu["matches"].To.tolist()[:4] == ["sitting", "Joan Smyth", "Microsoft", "apple"]      # a tie: the lower index
