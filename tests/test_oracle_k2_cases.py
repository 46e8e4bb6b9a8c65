"""CPU checks of the K2 tie / threshold case generators (tests/k2_cases.py) and of the oracle they are judged by: the runs
sit where the generators say, the thresholds are attained scores, and oracle/spdot_topn.c agrees with a plain Python
statement of the contract (explicit loops, products rounded, ascending terms, strict >, key (score desc, index asc))."""
import math

import numpy as np
import pytest
import scipy.sparse as sp

import k2_cases as kc
from oracle import native as onative
from oracle import tfidf as otfidf
from polyfuzz_b200.distributed import shard_bounds


@pytest.fixture(scope="module")
def case():
    return kc.TieCase()


@pytest.fixture(scope="module")
def vectors(case):
    return {mode: kc.canonical_vectors(case, mode) for mode in ("two", "self")}


@pytest.fixture(scope="module")
def lists0(vectors):
    out = {}
    for mode, (f, t) in vectors.items():
        out[mode] = onative.spdot_topn(f, t, kc.K_MAX, 0.0, self_match=mode == "self", n_threads=8)
    return out


def _straddles(pos, b):
    return any(p < b for p in pos) and any(p >= b for p in pos)


def test_runs_straddle_tile_split_and_shard_boundaries(case):
    for f, pos in enumerate(case.run_pos):
        assert all(case.to[p] == case.base[f] for p in pos)
        assert sum(s == case.base[f] for s in case.to) == len(pos)
        assert len(pos) > kc.K_MAX                          # longer than any list: every rank of B_f's list is in the run
        for variant, tiles in kc.TILES.items():
            for t in tiles:
                if t is None:
                    continue
                tile = kc.index_tile("block" if variant.startswith("block") else variant, case.n_to, t,
                                     32 if variant == "block32" else 16)
                nt = kc.n_tiles_of(case.n_to, tile)
                if tile <= 1024:
                    for q in range(1, nt):
                        if q * tile < 1024 or tile >= 256:
                            assert {q * tile - 1 - f, q * tile + f} <= set(pos), (variant, tile, q)
                for b in kc.split_starts(nt, 2, tile):
                    assert _straddles(pos, b) and {b - 1 - f, b + f} <= set(pos)
        for g in kc.SHARDS:
            for r in range(1, g):
                lo = shard_bounds(case.n_to, g, r)[0]
                assert {lo - 1 - f, lo + f} <= set(pos)


def test_word_pairs_share_a_16_bit_accumulator_word(case):
    pairs = list(zip(case.word_pos[::2], case.word_pos[1::2]))
    for t in kc.WORD_TILES:
        assert kc.index_tile("block", case.n_to, t, 16) == t
        mine = [(j, j2) for j, j2 in pairs if j2 - j == t // 2 and j // t == j2 // t]
        assert len(mine) >= 1
        for j, j2 in mine:
            assert j % t < t // 2 and j2 % t == j % t + t // 2      # the two cells of word j % t
    assert all(case.to[p] == case.word for p in case.word_pos)


def test_runs_cross_the_page_boundaries(case, lists0):
    oi, ov = lists0["two"]
    for f, h in enumerate(kc.HEADS):
        r = case.frm.index(case.var[f])
        heads, run = case.head_pos[f], case.run_pos[f]
        assert sorted(oi[r, :h].tolist()) == heads                  # V_f's copies first ...
        assert oi[r, h:].tolist() == run[:kc.K_MAX - h]             # ... then the run of B_f, in index order
        s = kc.run_score(oi, ov, r, run)
        assert (ov[r, h:] == s).all() and (ov[r, :h] > s).all()
        for page_end in (32, 64):
            if h < page_end < kc.K_MAX:                             # ranks page_end - 1 and page_end are both in the run
                assert oi[r, page_end - 1] in run and oi[r, page_end] in run


def test_identical_from_rows(case, lists0, vectors):
    for mode in ("two", "self"):
        rows = case.identical_from_rows(mode)
        assert len(rows) == kc.N_IDENTICAL_FROM > 16
        oi, ov = lists0[mode]
        f, _ = vectors[mode]
        ss = kc.self_scores(f[rows[:1]])[0]
        for k in kc.KS:
            kc.assert_identical_rows_agree(oi[:, :k], ov[:, :k], rows, mode == "self", k, self_score=ss)


def test_thresholds_are_attained_and_their_neighbours_are_not(case, lists0):
    for mode in ("two", "self"):
        oi, ov = lists0[mode]
        runs = [kc.run_score(oi, ov, case.from_list(mode).index(case.var[f]), case.run_pos[f]) for f in range(len(kc.HEADS))]
        base, ths = kc.thresholds(oi, ov, runs)
        got = set(ov[oi >= 0].tolist())
        for v in base:
            assert v in got
            assert math.nextafter(v, -math.inf) not in got and math.nextafter(v, math.inf) not in got
        assert 1.0 in got and any(1.0 < x < 1.0 + 1e-15 for x in got)
        assert -0.5 in ths and 1.0 in ths and math.nextafter(1.0, 0.0) in ths


def test_exact_one_and_above_one_pairs_exist(case, vectors, lists0):
    for mode in ("two", "self"):
        f, t = vectors[mode]
        src = case.from_list(mode)
        for s in case.ones:                                          # single n-gram rows: weight exactly 1.0
            r = src.index(s)
            assert f.indptr[r + 1] - f.indptr[r] == 1 and f.data[f.indptr[r]] == 1.0
        oi, ov = lists0[mode]
        r = src.index("aaa")
        assert ov[r, 0] == 1.0
        ss = kc.self_scores(t)
        above = [s for s in case.dups if ss[case.to.index(s)] > 1.0]
        assert above, "no duplicated string scores above 1.0 with its copy"
        r = src.index(above[0])
        assert 1.0 < ov[r, 0] < 1.0 + 1e-15                       # above 1.0 by an ulp or two


@pytest.mark.parametrize("n,seed", [(128, 1), (129, 2), (256, 3), (257, 4)])
def test_distinct_trigram_rows(n, seed):
    s = kc.distinct_trigram_string(n, seed)
    o = otfidf.TfidfOracle().fit([s, "abc def"])
    m = o.transform([s])
    assert m.indptr[1] == n and len(set(otfidf.create_ngrams(s))) == n


@pytest.mark.parametrize("slots,rng", [(8192, (3, 3)), (8193, (3, 3)), (8193, (3, 4))])
def test_slot_count_strings(slots, rng):
    s = kc.string_with_slots(slots, rng)
    from polyfuzz_b200.strings import ngram_slot_bounds
    offs = np.array([0, len(s)], dtype=np.int64)
    got, _ = ngram_slot_bounds(offs, *rng)
    assert int(got[0]) == slots


def test_slot_count_that_no_length_gives_is_refused():
    with pytest.raises(ValueError):
        kc.string_with_slots(8192, (3, 4))                  # 2 * len - 5 is odd


# ---- the oracle against a plain statement of the contract -------------------------------------------------------------
def py_spdot_topn(a, b, k, lb, self_match=False, from_base=0, to_base=0):
    a = sp.csr_matrix(a); b = sp.csr_matrix(b)
    idx = np.full((a.shape[0], k), -1, dtype=np.int32); val = np.zeros((a.shape[0], k))
    for i in range(a.shape[0]):
        ra = dict(zip(a.indices[a.indptr[i]:a.indptr[i + 1]].tolist(), a.data[a.indptr[i]:a.indptr[i + 1]].tolist()))
        cands = []
        for j in range(b.shape[0]):
            cols = b.indices[b.indptr[j]:b.indptr[j + 1]].tolist()
            vals = b.data[b.indptr[j]:b.indptr[j + 1]].tolist()
            s, touched = 0.0, False
            for c, w in sorted(zip(cols, vals)):                     # ascending term
                if c in ra:
                    p = ra[c] * w                                    # product rounded ...
                    s = s + p                                        # ... then added
                    touched = True
            if not touched or not s > lb:
                continue
            if self_match and to_base + j == from_base + i:
                continue
            cands.append((s, to_base + j))
        cands.sort(key=lambda t: (-t[0], t[1]))
        for r, (s, j) in enumerate(cands[:k]):
            idx[i, r] = j; val[i, r] = s
    return idx, val


@pytest.fixture(scope="module")
def small_pairs():
    from polyfuzz_b200 import synth
    names = synth.company_names(60, seed=5)
    to = names[:30] + [names[3]] * 4 + ["aaa", "aaaa"] + names[40:50]
    frm = names[25:45] + [names[3], "aaa", "", "zz"]
    f, t, _ = otfidf.fit_transform_sklearn(frm, to)
    return f, t


def test_oracle_matches_python_statement(small_pairs):
    f, t = small_pairs
    oi, ov = onative.spdot_topn(f, t, 12, 0.0)
    scores = sorted(set(ov[oi >= 0].tolist()))
    vals, cnt = np.unique(ov[oi >= 0], return_counts=True)
    ths = {0.0, -0.5, 1.0, math.nextafter(1.0, 0.0), scores[len(scores) // 2], float(vals[np.argmax(cnt)])}
    ths |= {math.nextafter(x, d) for x in list(ths) for d in (-math.inf, math.inf)}
    for lb in sorted(ths):
        for k in (1, 5, 12):
            pi, pv = py_spdot_topn(f, t, k, lb)
            ci, cv = onative.spdot_topn(f, t, k, lb)
            np.testing.assert_array_equal(ci, pi, err_msg=f"lb={lb!r} k={k}")
            np.testing.assert_array_equal(cv, pv, err_msg=f"lb={lb!r} k={k}")


def test_oracle_self_match_with_bases_matches_python_statement(small_pairs):
    _, t = small_pairs
    n = t.shape[0]
    for lo, hi, tlo, thi in ((0, n, 0, n), (10, 30, 0, n), (10, 30, 20, n), (5, 25, 0, 18)):
        a, b = t[lo:hi], t[tlo:thi]
        ref = onative.spdot_topn(t, t, 6, 0.0, self_match=True)
        lbs = sorted({0.0, float(np.median(ref[1][ref[0] >= 0])), 1.0})
        for lb in lbs + [math.nextafter(x, -math.inf) for x in lbs]:
            pi, pv = py_spdot_topn(a, b, 6, lb, True, lo, tlo)
            ci, cv = onative.spdot_topn(a, b, 6, lb, self_match=True, from_index_base=lo, to_index_base=tlo)
            np.testing.assert_array_equal(ci, pi)
            np.testing.assert_array_equal(cv, pv)


def py_topk_merge(idx, val, k_out):
    G, n, k_in = idx.shape
    oi = np.full((n, k_out), -1, dtype=np.int32); ov = np.zeros((n, k_out))
    for i in range(n):
        c = [(float(val[g, i, r]), int(idx[g, i, r])) for g in range(G) for r in range(k_in) if idx[g, i, r] >= 0]
        c.sort(key=lambda t: (-t[0], t[1]))
        for r, (s, j) in enumerate(c[:k_out]):
            oi[i, r] = j; ov[i, r] = s
    return oi, ov


@pytest.mark.parametrize("n_lists,k_in,k_out", [(3, 5, 7), (2, 40, 33), (4, 12, 32), (1, 70, 70), (3, 33, 5)])
def test_oracle_topk_merge_matches_python_statement(n_lists, k_in, k_out):
    idx, val = kc.crafted_merge_lists(n_lists, 40, k_in, seed=k_in + k_out)
    ci, cv = onative.topk_merge(idx, val, k_out)
    pi, pv = py_topk_merge(idx, val, k_out)
    np.testing.assert_array_equal(ci, pi)
    np.testing.assert_array_equal(cv, pv)
