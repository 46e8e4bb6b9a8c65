"""GPU parity tests of K3b on long strings: from-strings of 256..1 024 code points (the 4-, 8- and 16-word classes, the last
two one CTA per from-row) and to-strings of any length, against oracle/fuzz.py (rapidfuzz 3.x restated).  Indices and scores
are compared with ==.  oracle.fuzz.lcs_len is swapped for the textbook C LCS of tests/lcs_oracle.c in this module only."""
import numpy as np
import pytest

import lcs_oracle
from oracle import fuzz as ofuzz

pytestmark = pytest.mark.gpu

SCORERS = ["WRatio", "QRatio", "partial_ratio", "token_sort_ratio", "token_set_ratio", "token_ratio",
           "partial_token_sort_ratio", "partial_token_set_ratio", "partial_token_ratio", "ratio"]
WORDS = ["The", "of", "and", "a", "Night", "Day", "Love", "Man", "Last", "Story", "Dead", "II", "Return", "King", "night", "é",
         "Noël", "x", "Zorro", "Christmas", "Carol", "day", "man", "House", "Home", "Street", "Road", "Avenue", "North", "12",
         "34b", "Suite", "Unit", "Floor", "Building", "Park", "Lane", "West", "East", "Apt"]


@pytest.fixture(scope="module", autouse=True)
def c_lcs():
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ofuzz, "lcs_len", lcs_oracle.lcs_len)
        yield


@pytest.fixture(scope="module")
def fz():
    from polyfuzz_b200 import fuzzy
    return fuzzy


def text(rng, n, words=WORDS):
    """Whitespace-separated words, exactly n code points, no leading / trailing space (so |S(s)| = |U(s)| bound = n)."""
    out = ""
    while len(out) < n:
        out += (" " if out else "") + str(rng.choice(words))
    out = out[:n]
    return out[:-1] + "y" if out.endswith(" ") else out


def titles(rng, n, lo=1, hi=8):
    return [" ".join(rng.choice(WORDS, rng.integers(lo, hi + 1))) for _ in range(n)]


def score_matrix(frm, to, scorer, cutoff=0.0):
    fn = ofuzz.SCORERS[scorer]
    return np.array([[fn(a, b, cutoff) for b in to] for a in frm], dtype=np.float64)


def oracle_topk(S, k, cutoff=0.0, exclude_self=False):
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
    np.testing.assert_array_equal(got[0].cpu().numpy(), exp[0])
    np.testing.assert_array_equal(got[1].cpu().numpy(), exp[1])


def check(fz, frm, to, scorer, S, cutoff=0.0, exclude_self=False, ks=(2, 10, 32), splits=(1, 3, None)):
    """arg-best and top-k at every k and split count against the oracle matrix S (scored at the same cutoff)"""
    for n_splits in splits:
        bi, bs = fz.fuzz_argbest(frm, to, scorer, cutoff, exclude_self=exclude_self, n_splits=n_splits)
        ei, ev = oracle_topk(S, 1, cutoff, exclude_self)
        _eq((bi, bs), (ei[:, 0], ev[:, 0]))
        for k in ks:
            _eq(fz.fuzz_topk(frm, to, k, scorer, cutoff, exclude_self=exclude_self, n_splits=n_splits),
                oracle_topk(S, k, cutoff, exclude_self))


# ---- every scorer across the word-class boundaries --------------------------------------------------------------------------
FROM_LENS = (255, 256, 257, 511, 512, 513, 1023, 1024)
_GRID = {}


def grid():
    """from-strings at both sides of every class boundary (plus two short ones); to-strings: titles, and 200 / 257 / 300 code
    points, so the partial scorers see a shorter, a longer and an equally long to-string (the swap of partial_ratio)."""
    if not _GRID:
        rng = np.random.default_rng(20261016)
        frm = [text(rng, n) for n in FROM_LENS] + [text(rng, 30), text(rng, 100)]
        to = titles(rng, 40) + [text(rng, 200), text(rng, 257), text(rng, 300), frm[2][:150] + " Zorro " + frm[2][157:],
                                frm[4][:300], ""]
        _GRID.update(frm=frm, to=to)
    return _GRID["frm"], _GRID["to"]


@pytest.mark.parametrize("scorer", SCORERS)
def test_every_scorer_across_word_classes(fz, scorer):
    frm, to = grid()
    check(fz, frm, to, scorer, score_matrix(frm, to, scorer))


# ---- to-strings of 1 500 and 5 000 code points ----------------------------------------------------------------------------
@pytest.mark.parametrize("scorer", ["WRatio", "partial_ratio", "token_set_ratio", "partial_token_ratio"])
def test_long_to_strings(fz, scorer):
    rng = np.random.default_rng(7)
    frm = [text(rng, 40), text(rng, 150), text(rng, 300)]
    to = titles(rng, 20) + [text(rng, 1500), text(rng, 5000), frm[2] + " " + text(rng, 1200)]
    check(fz, frm, to, scorer, score_matrix(frm, to, scorer), ks=(2, 32), splits=(1, None))


@pytest.mark.parametrize("scorer", ["WRatio", "partial_ratio"])
def test_from_1024_against_1500(fz, scorer):
    rng = np.random.default_rng(8)
    frm = [text(rng, 1024), text(rng, 1000)]
    to = titles(rng, 10) + [text(rng, 1500)]
    check(fz, frm, to, scorer, score_matrix(frm, to, scorer), ks=(2,), splits=(None,))


# ---- token_set_ratio: joined differences past 255 on each side and past 1 024 on the to-side --------------------------------
def _vocab(rng, prefix, n):
    return [prefix + "".join(rng.choice(list("abcdefghijklmnop"), rng.integers(2, 8))) for _ in range(n)]


@pytest.mark.parametrize("scorer", ["token_set_ratio", "token_ratio", "WRatio", "partial_token_set_ratio"])
def test_token_set_long_differences(fz, scorer):
    rng = np.random.default_rng(3)
    A, B = _vocab(rng, "a", 150), _vocab(rng, "b", 150)
    common = ["Common", "Shared"]
    frm = [text(rng, 1000, A + common) + " Common", text(rng, 700, A + B) + " Shared", text(rng, 400, A)]
    distinct = []                                              # distinct words, each once: U(b) is as long as b
    while len(" ".join(distinct)) <= 1100:
        w = _vocab(rng, "c", 1)[0]
        if w not in distinct:
            distinct.append(w)
    to = [text(rng, 1400, B + common) + " Common", text(rng, 900, B + A) + " Shared", text(rng, 500, B), "Common Shared",
          text(rng, 1100, A + B + common), " ".join(distinct) + " Common"]
    diff = lambda a, b: len(" ".join(sorted(set(a.split()) - set(b.split()))))
    assert "Common" in frm[0].split() and diff(to[-1], frm[0]) > 1024 and diff(frm[0], to[-1]) > 255
    S = score_matrix(frm, to, scorer)
    check(fz, frm, to, scorer, S, ks=(2, 5), splits=(1, None))
    for c in (40.0, 70.0):                                    # the cutoff threads through the differences' distance
        check(fz, frm, to, scorer, score_matrix(frm, to, scorer, c), cutoff=c, ks=(3,), splits=(None,))


# ---- one CTA per row: every warp takes several to-groups of one split before the merge -----------------------------------------
@pytest.mark.parametrize("scorer", ["WRatio", "token_set_ratio", "partial_ratio"])
def test_cta_rows_over_many_groups(fz, scorer):
    rng = np.random.default_rng(23)
    frm = [text(rng, 600), text(rng, 1000), text(rng, 300), text(rng, 257)]
    to = titles(rng, 400) + [frm[0][:450], frm[1][:800]]                   # 13 groups of 32: 3-4 per warp at n_splits=1
    check(fz, frm, to, scorer, score_matrix(frm, to, scorer), ks=(5, 32), splits=(1,))


# ---- non-ASCII, and more than 254 distinct code points over the from-list (alphabet batches) ---------------------------------
def test_non_ascii_and_alphabet_batches(fz):
    rng = np.random.default_rng(5)
    blocks = [[chr(0x4E00 + 97 * b + i) for i in range(60)] for b in range(6)]
    frm = [" ".join("".join(rng.choice(bl, rng.integers(1, 6))) for _ in range(300))[:n] for bl, n in zip(blocks, (300, 520, 700, 260, 900, 1024))]
    frm = [s.strip() for s in frm]
    assert len(set("".join(frm))) > 255
    pool = [c for bl in blocks for c in bl] + list("éNoëlxyz")
    to = [" ".join("".join(rng.choice(pool, rng.integers(1, 5))) for _ in range(rng.integers(2, 12))) for _ in range(30)]
    to += [frm[1][:200] + " éé " + frm[1][204:], frm[5][100:400], " ".join(frm[3].split()[::-1])]
    for scorer in ("WRatio", "token_set_ratio", "partial_ratio", "token_sort_ratio"):
        check(fz, frm, to, scorer, score_matrix(frm, to, scorer), ks=(4,), splits=(None,))


# ---- self-match with a cutoff ------------------------------------------------------------------------------------------------
def _family(rng, n):
    """n long strings that share most of their words: a base text with words swapped, dropped and appended"""
    base = text(rng, 400).split()
    out = []
    for _ in range(n):
        w = [x if rng.random() > 0.2 else str(rng.choice(WORDS)) for x in base if rng.random() > 0.1]
        w += list(rng.choice(WORDS, rng.integers(0, 60)))
        out.append(" ".join(w)[:rng.integers(260, 1025)].strip())
    return out


@pytest.mark.parametrize("scorer,cutoff", [("WRatio", 60.0), ("token_set_ratio", 50.0), ("token_ratio", 70.0)])
def test_self_match_with_cutoff(fz, scorer, cutoff):
    rng = np.random.default_rng(11)
    names = _family(rng, 10)
    names.append(names[3])                                     # a duplicate: its best match is its twin at 100
    S = score_matrix(names, names, scorer, cutoff)
    check(fz, names, names, scorer, S, cutoff=cutoff, exclude_self=True, ks=(3,), splits=(1, None))
    bi, _ = fz.fuzz_argbest(names, names, scorer, cutoff, exclude_self=True)
    assert (bi.cpu().numpy() != np.arange(len(names))).all()


# ---- short and long from-strings in one list ---------------------------------------------------------------------------------
def test_mixed_short_and_long_rows(fz):
    rng = np.random.default_rng(13)
    long_ = [text(rng, 300), text(rng, 600), text(rng, 1000)]
    frm = titles(rng, 30)[:15] + long_ + titles(rng, 30)[:15]
    to = titles(rng, 120) + [long_[0][:280], text(rng, 800)]
    for scorer in ("WRatio", "token_set_ratio"):
        S = score_matrix(frm, to, scorer)
        check(fz, frm, to, scorer, S, ks=(5,), splits=(None,))
        # the short rows alone give the same answers as in the mixed call
        short = [i for i in range(len(frm)) if len(frm[i]) <= 256]
        bi, bs = fz.fuzz_argbest([frm[i] for i in short], to, scorer)
        ei, ev = oracle_topk(S[short], 1)
        _eq((bi, bs), (ei[:, 0], ev[:, 0]))


# ---- the matcher frames --------------------------------------------------------------------------------------------------------
def test_matchers_on_long_strings():
    from polyfuzz_b200 import EditDistance, RapidFuzz
    rng = np.random.default_rng(17)
    frm = [text(rng, 700), text(rng, 300), "Night of the Living Dead"]
    to = titles(rng, 25) + [frm[0][:500], text(rng, 1200), frm[1] + " II"]
    S = score_matrix(frm, to, "WRatio")
    ei, ev = oracle_topk(S, 2)
    m = RapidFuzz().match(frm, to)
    assert m.To.tolist() == [to[j] for j in ei[:, 0]] and m.Similarity.tolist() == (ev[:, 0] / 100).tolist()
    m = RapidFuzz(top_n=2).match(frm, to)
    assert m.To_2.tolist() == [to[j] for j in ei[:, 1]] and m.Similarity_2.tolist() == (ev[:, 1] / 100).tolist()
    S = score_matrix(frm, to, "token_set_ratio")
    ei, ev = oracle_topk(S, 1)
    e = EditDistance(scorer="token_set_ratio", normalize=False).match(frm, to)
    assert e.To.tolist() == [to[j] for j in ei[:, 0]] and e.Similarity.tolist() == ev[:, 0].tolist()


# ---- distributed=True: per-shard calls merged ------------------------------------------------------------------------------------
def test_to_shards_merge_equals_single_call(fz):
    import torch
    from polyfuzz_b200.distributed import merge_topk_any, shard_bounds
    rng = np.random.default_rng(19)
    s = _family(rng, 8) + titles(rng, 6)
    whole = fz.fuzz_topk(s, s, 4, "WRatio", 50.0, exclude_self=True)
    parts = []
    for r in range(2):
        lo, hi = shard_bounds(len(s), 2, r)
        parts.append(fz.fuzz_topk(s, s[lo:hi], 4, "WRatio", 50.0, exclude_self=True, self_shift=-lo, to_index_base=lo))
    merged = merge_topk_any(torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts]), 4)
    for a, b in zip(whole, merged):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    _eq(merged, oracle_topk(score_matrix(s, s, "WRatio", 50.0), 4, 50.0, exclude_self=True))


def test_from_string_over_1024_code_points_is_refused(fz):
    with pytest.raises(ValueError, match="at most 1024"):
        fz.fuzz_argbest(["a" * 1025], ["a"], "WRatio")
    bi, bs = fz.fuzz_argbest(["a" * 1024], ["b", "a" * 6000], "partial_ratio")
    assert int(bi[0]) == 1 and float(bs[0]) == 100.0
