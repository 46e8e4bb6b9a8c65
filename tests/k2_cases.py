"""Case generators for the K2 tie and threshold tests (TEST INFRASTRUCTURE, NOT PRODUCT CODE; no GPU needed).

Every input is a string list that goes through the real vectoriser, so every row is an l2-normalised TF-IDF row as in
production.  Ties are exact by construction: identical to-strings give bit-identical to-rows, so a from-row scores all of
them bit-identically under the canonical order (fp64, ascending terms, product rounded before the add).  The runs of
identical strings are placed on the boundaries where the K2 kernels hand a tied run from one piece of work to the next:
to-tiles, tile splits (`tiles_per = ceil(n_tiles / n_splits)`), to-shards (`distributed.shard_bounds`), the two cells of a
16-bit block accumulator word (to-rows j and j + tile/2) and the 32-entry pages of top_n > 32."""
import math

import numpy as np

from polyfuzz_b200 import synth
from polyfuzz_b200.distributed import shard_bounds

N_TO = 6000
HEADS = (5, 30, 62)            # copies of V_f ranked ahead of the run of B_f for from-row V_f: the run then covers ranks
                               # 5.., 30.. and 62.., so it crosses the page boundaries 31/32 and 63/64
N_IDENTICAL_FROM = 17          # identical from-rows: more than the largest block (16 rows), so they straddle a block boundary
KS = (1, 7, 32, 33, 64, 70)
K_MAX = max(KS)

# the smallest legal tile of each index variant, and the larger ones the tests use (None: the variant's default)
TILES = {"list": (64, 512), "dense": (64, 1024), "dense32": (64, 1024), "block16": (256, 1024, None), "block32": (128, 1024, None),
         "hash": (64, 1024, None)}
WORD_TILES = (256, 1024, 4096)  # 16-bit block tiles whose word pairs (j, j + tile/2) hold a tied pair
SHARDS = (2, 3)


def index_tile(variant, n_to, tile=None, acc_bits=16):
    """The tile engine.SparseIndex builds (the GPU tests assert that the real index agrees): requested tile clipped to
    64 .. round_up(n_to, 64); block tiles rounded up to the 128-word scan step and capped at 4 096."""
    default = {"list": 512, "dense": 1024, "dense32": 1024, "block": 4096, "hash": 65536}
    if tile is None:
        tile = default[variant]
        if variant == "block" and acc_bits != 16:
            tile //= 2
    tile = max(64, min(int(tile), ((max(n_to, 1) + 63) // 64) * 64))
    if variant == "block":
        step = 128 * (2 if acc_bits == 16 else 1)
        tile = min(4096, max(step, (tile + step - 1) // step * step))
    return tile


def n_tiles_of(n_to, tile):
    return max(1, (n_to + tile - 1) // tile)


def split_starts(n_tiles, n_splits, tile):
    """First to-row of every tile split after the first (the kernels' rule: tiles_per = ceil(n_tiles / n_splits))."""
    per = (n_tiles + n_splits - 1) // n_splits
    return [s * per * tile for s in range(1, n_splits) if s * per < n_tiles]


def boundaries(n_to=N_TO):
    """To-rows where one piece of K2 work ends and the next begins: tile starts of tiles 64 .. 1 024 (64 and 128 in the
    first 1 024 rows only, to keep the runs short), the starts of the second split of every tile at n_splits = 2, and the
    shard starts for 2 and 3 shards."""
    b = set()
    for t in (64, 128):
        b.update(range(t, min(n_to, 1024), t))
    for t in (256, 512, 1024):
        b.update(range(t, n_to, t))
    for t in sorted({v for ts in TILES.values() for v in ts if v is not None}):
        b.update(split_starts(n_tiles_of(n_to, t), 2, t))
    for g in SHARDS:
        b.update(shard_bounds(n_to, g, r)[0] for r in range(1, g))
    return sorted(x for x in b if 3 <= x <= n_to - 3)


def _family_strings(n):
    """n unrelated base strings B_f (a name plus a rare token) and their longer variants V_f = B_f + ' zyx'."""
    names = synth.company_names(n, seed=901)
    base = [f"{s} qx{f}vk" for f, s in enumerate(names)]
    return base, [b + " zyxw" for b in base]


class TieCase:
    """to / from lists with tied runs on the boundaries, and what was placed where.

    run_pos[f]   to-rows holding B_f (two per boundary: b - 1 - f and b + f)
    head_pos[f]  to-rows holding V_f (HEADS[f] copies)
    word_pos     to-rows holding W: pairs (j, j + tile/2) inside tiles of WORD_TILES
    ident        the string of the N_IDENTICAL_FROM identical from-rows (also in the to-list for the self-match)
    ones         single-n-gram strings: every weight is exactly 1.0 and they score exactly 1.0 with each other
    dups         strings put twice into both lists (some of them score above 1.0 with their copy)"""

    def __init__(self, n_to=N_TO, seed=3):
        rng = np.random.default_rng(seed)
        self.n_to = n_to
        fill = synth.company_names(n_to, seed=seed)
        taken = set()
        self.base, self.var = _family_strings(len(HEADS))
        bnd = boundaries(n_to)
        self.run_pos = []
        for f in range(len(HEADS)):
            pos = sorted({b - 1 - f for b in bnd} | {b + f for b in bnd})
            pos = [p for p in pos if p not in taken]
            taken.update(pos)
            self.run_pos.append(pos)
        self.word = "wordpair kelvinator qz7j"
        self.word_pos = []
        for w, t in enumerate(WORD_TILES):
            for q in range(n_tiles_of(n_to, t)):
                j = q * t + 11 + 3 * w
                if j + t // 2 < n_to and j not in taken and j + t // 2 not in taken:
                    self.word_pos += [j, j + t // 2]
                    taken.update((j, j + t // 2))
        free = np.array(sorted(set(range(n_to)) - taken))
        picks = rng.permutation(free)
        c = 0
        self.head_pos = []
        for h in HEADS:
            self.head_pos.append(sorted(int(x) for x in picks[c:c + h])); c += h
        self.ident = "identical rows llc qv"
        self.ident_pos = sorted(int(x) for x in picks[c:c + N_IDENTICAL_FROM]); c += N_IDENTICAL_FROM
        self.ones = ["aaa", "aaaa", "bbb", "bbbbb", "aaa"]
        self.ones_pos = sorted(int(x) for x in picks[c:c + len(self.ones)]); c += len(self.ones)
        self.dups = synth.company_names(12, seed=977)
        self.dup_pos = [int(x) for x in picks[c:c + 2 * len(self.dups)]]; c += 2 * len(self.dups)
        to = list(fill)
        for f in range(len(HEADS)):
            for p in self.run_pos[f]:
                to[p] = self.base[f]
            for p in self.head_pos[f]:
                to[p] = self.var[f]
        for p in self.word_pos:
            to[p] = self.word
        for p in self.ident_pos:
            to[p] = self.ident
        for p, s in zip(self.ones_pos, self.ones):
            to[p] = s
        for q, p in enumerate(self.dup_pos):
            to[p] = self.dups[q // 2]
        self.to = to
        frm = list(self.base) + list(self.var) + [self.word] + [self.ident] * N_IDENTICAL_FROM + list(self.ones)
        frm += self.dups + self.dups + synth.company_names(700, seed=seed + 1000) + [to[17], to[4000], "", "zz"]
        order = np.random.default_rng(seed + 1).permutation(len(frm))
        self.frm = [frm[i] for i in order]

    # ---- what the from-lists of each mode are -----------------------------------------------------------------------
    def from_list(self, mode):
        return self.to if mode == "self" else self.frm

    def identical_from_rows(self, mode):
        src = self.from_list(mode)
        return [i for i, s in enumerate(src) if s == self.ident]


def canonical_vectors(case, mode):
    """(from CSR, to CSR) through the oracle vectoriser: two lists are fitted together, a self-match on the to-list alone."""
    from oracle import tfidf as otfidf
    if mode == "self":
        _, t, _ = otfidf.fit_transform_sklearn(case.to, None)
        return t, t
    f, t, _ = otfidf.fit_transform_sklearn(case.frm, case.to)
    return f, t


def self_scores(m):
    """Canonical score of every row with itself (an identical copy of it scores the same)."""
    out = np.zeros(m.shape[0])
    for i in range(m.shape[0]):
        s = 0.0
        for x in m.data[m.indptr[i]:m.indptr[i + 1]]:
            s = s + x * x
        out[i] = s
    return out


def run_score(oi, ov, row, members):
    """The score row gives the run `members` (all identical to-rows), read from its list."""
    hit = np.isin(oi[row], members)
    assert hit.any(), "the run is not in the row's list"
    vals = np.unique(ov[row][hit])
    assert len(vals) == 1, "a run of identical to-rows must score identically"
    return float(vals[0])


def thresholds(oi, ov, run_scores):
    """min_similarity values on attained scores, from the ms = 0 lists (oi, ov): every run score, the most frequent and
    the median score below 0.999, and the doubles just below and above each; 1.0 and the double below it; a negative
    value."""
    got = ov[oi >= 0]
    vals, cnt = np.unique(got[got < 0.999], return_counts=True)       # (the duplicates' scores next to 1.0 have 1.0 of their own)
    frequent = float(vals[np.argmax(cnt)])
    median = float(np.sort(got)[len(got) // 2])
    if median >= 0.999:
        median = float(np.sort(got[got < 0.999])[(got < 0.999).sum() // 2])
    base = sorted(set(run_scores) | {frequent, median})
    out = []
    for v in base:
        out += [math.nextafter(v, -math.inf), v, math.nextafter(v, math.inf)]
    out += [1.0, math.nextafter(1.0, 0.0), -0.5]
    return base, sorted(set(out))


def complete_list(idx, val, row, self_idx, self_score, k):
    """A self-match list with the diagonal put back at its canonical place: identical from-rows must give the same."""
    items = [(float(v), int(j)) for j, v in zip(idx[row], val[row]) if j >= 0]
    items.append((self_score, self_idx))
    items.sort(key=lambda t: (-t[0], t[1]))
    return items[:k]


def assert_identical_rows_agree(idx, val, rows, self_match, k, self_base=0, self_score=None):
    """Identical from-rows get identical lists (in a self-match: identical once each row's diagonal is put back)."""
    if self_match:
        ref = complete_list(idx, val, rows[0], self_base + rows[0], self_score, k)
        for r in rows[1:]:
            assert complete_list(idx, val, r, self_base + r, self_score, k) == ref, f"identical from-row {r} differs"
    else:
        for r in rows[1:]:
            assert np.array_equal(idx[r], idx[rows[0]]) and np.array_equal(val[r], val[rows[0]]), f"identical from-row {r} differs"


# ---- row sizes ----------------------------------------------------------------------------------------------------
def distinct_trigram_string(n, seed):
    """A string over [a-z0-9] with exactly n trigrams, all distinct (length n + 2; no spaces, nothing the cleaner drops)."""
    rng = np.random.default_rng(seed)
    alpha = "abcdefghijklmnopqrstuvwxyz0123456789"
    s = "".join(rng.choice(list(alpha), 2))
    seen = set()
    while len(s) < n + 2:
        for c in rng.permutation(list(alpha)):
            g = s[-2:] + c
            if g not in seen:
                seen.add(g); s += c
                break
        else:
            raise RuntimeError("dead end")
    return s


def slot_count(length, ngram_range):
    lo, hi = ngram_range
    return sum(max(0, length - n + 1) for n in range(lo, hi + 1))


def string_with_slots(n_slots, ngram_range, seed=0):
    """A uniform [a-z0-9 ] string whose n-gram slot count (sum over n of len - n + 1, the vectoriser's per-string bound)
    is exactly n_slots."""
    for length in range(1, 4 * n_slots + 16):
        if slot_count(length, ngram_range) == n_slots:
            return synth.uniform_strings(1, seed=seed, lo=length, hi=length)[0]
        if slot_count(length, ngram_range) > n_slots:
            break
    raise ValueError(f"no string length gives {n_slots} slots for range {ngram_range}")


# ---- merges -------------------------------------------------------------------------------------------------------
def crafted_merge_lists(n_lists, n_from, k_in, seed, n_scores=3, p_empty=0.25):
    """[n_lists, n_from, k_in] candidate lists with few distinct scores (ties across lists), empty slots (-1, 0.0) at
    random positions, and to-indices that are unique per row and unordered across lists."""
    rng = np.random.default_rng(seed)
    scores = np.sort(rng.random(n_scores))[::-1]
    idx = np.full((n_lists, n_from, k_in), -1, dtype=np.int32)
    val = np.zeros((n_lists, n_from, k_in), dtype=np.float64)
    for i in range(n_from):
        js = rng.permutation(10 * n_lists * k_in)[:n_lists * k_in].reshape(n_lists, k_in)
        for l in range(n_lists):
            v = np.sort(rng.choice(scores, k_in))[::-1]
            order = np.lexsort((js[l], -v))                 # each list in canonical order, as the kernels hand them over
            idx[l, i] = js[l][order]; val[l, i] = v[order]
            empty = rng.random(k_in) < p_empty
            if i % 7 == 0:
                empty[:] = True                             # a list with nothing in it
            idx[l, i][empty] = -1; val[l, i][empty] = 0.0
    return idx, val
