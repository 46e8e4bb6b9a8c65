"""K3 host driver: all-pairs edit distance with per-row arg-best on the GPU (include/pfz.h, pfz_lev_rows).

Semantics restated from the reference's call sites (polyfuzz/models/_rapidfuzz.py:99-113,
polyfuzz/models/_distance.py:89-102) and rapidfuzz's published definitions:
    "ratio"     fuzz.ratio           = (1 - indel/(|a|+|b|)) * 100            in [0, 100]
    "norm_lev"  Levenshtein.normalized_similarity = 1 - lev/max(|a|,|b|)       in [0, 1]
    "lev", "indel"  raw distances (best = smallest)
    "jaro"          jellyfish.jaro_similarity(from, to)                          in [0, 1]
    "jaro_winkler"  jellyfish.jaro_winkler_similarity(from, to), long_tolerance=False   in [0, 1]
    "norm_osa"  OSA.normalized_similarity = 1 - osa/max(|a|,|b|)               in [0, 1]
    "osa"       raw optimal string alignment distance (restricted Damerau-Levenshtein: adjacent swaps cost 1, no
                substring is edited twice, so osa("CA", "ABC") = 3 where unrestricted Damerau-Levenshtein gives 2)
    "norm_dl"   DamerauLevenshtein.normalized_similarity = 1 - dl/max(|a|,|b|)  in [0, 1]
    "dl"        raw unrestricted Damerau-Levenshtein distance (Lowrance-Wagner, unit costs: a swapped pair may be edited
                again, so dl("CA", "ABC") = 2); gated by an OSA pass (DESIGN.md 4.10)
    The sequence metrics, rapidfuzz 3.x's normalized_similarity = 1 - d/M (1.0 when M = 0), in [0, 1]; best_dist is d:
    "norm_indel"    Indel:   d = |a| + |b| - 2 LCS, M = |a| + |b|  (fuzz.ratio's ns, without its x100)
    "norm_lcsseq"   LCSseq:  d = M - LCS, M = max(|a|, |b|)
    "norm_hamming"  Hamming with pad=True (rapidfuzz 3's default; rapidfuzz 2 raises on unequal lengths): d = mismatches at the
                    positions both strings have + ||a| - |b||, M = max(|a|, |b|)
    "norm_prefix"   Prefix:  d = M - the common prefix length, M = max(|a|, |b|)
    "norm_postfix"  Postfix: d = M - the common suffix length, M = max(|a|, |b|)
    They take norm_lev's one-step cutoff (score >= score_cutoff) and have no distance matrix (DESIGN.md 4.18).
The Jaro metrics are computed on code points, from-string first (the reference calls scorer(from_string, to_string),
polyfuzz/models/_distance.py:98); their best_dist is the number of matching characters, and they have no distance
matrix (want_matrix=True raises ValueError).
Best match of a from-string = first to-string (lowest index) with the maximal score >= score_cutoff; the top-k functions
return the k best under the same key (score desc, index asc), k <= 32.

Two levels: `EditQueries` / `EditTargets` stage a from-list / to-list in HBM once (host packing, length sort,
alphabet batches); `edit_argbest_staged` only enqueues kernels, so a staged pair can be scored repeatedly
(bench.py's device-timed leg, the multi-GPU shards) without touching the host lists again.  `KeptTargets` holds a
matcher's last staged to-side, which a `re_train=False` call with an equal to-list scores against again.

Candidate mode (`edit_cand_topk_staged`, DESIGN.md 4.16): each from-row scores only the to-indices of its row of a device
int32 [n_from, c] candidate array (-1 = empty slot, distinct per row; TF-IDF's top-n), with the same kernels, scores, cutoffs
and key, so a row equals the all-pairs result against the to-strings of its list.

Weighted Levenshtein (`edit_wlev_argbest` / `edit_wlev_topk` / `edit_wlev_cand_topk` and their staged forms, pfz_wlev_rows,
DESIGN.md 4.17): rapidfuzz's Levenshtein.normalized_similarity(from, to, weights=(insertion, deletion, substitution)) = 1 - D/M
with norm_lev's key and cutoff, weights in [0, WLEV_MAX_WEIGHT].  Uniform weights (w, w, w) take the norm_lev path (the same
scores); it is not a METRIC (no raw distance, no matrix).  It uses the same EditQueries / EditTargets / KeptTargets.
"""
import numpy as np
import torch

from . import _lib
from .engine import _dev, _p, _stream, _to_dev, topk_merge
from .strings import pack_strings

METRIC = {"lev": 0, "indel": 1, "norm_lev": 2, "ratio": 3, "jaro": 4, "jaro_winkler": 5, "osa": 6, "norm_osa": 7, "dl": 8,
          "norm_dl": 9, "norm_indel": 11, "norm_lcsseq": 12, "norm_hamming": 13, "norm_prefix": 14, "norm_postfix": 15}
JARO_METRICS = ("jaro", "jaro_winkler")
SEQ_METRICS = ("norm_indel", "norm_lcsseq", "norm_hamming", "norm_prefix", "norm_postfix")
# DL metric -> the OSA metric whose k-th best score gates it (norm_osa <= norm_dl pair by pair, DESIGN.md 4.10)
DL_GATE = {"dl": "osa", "norm_dl": "norm_osa"}
N_CODE_POINTS = 0x110000
MAX_LEN = 1024


def _word_class(m):
    """n_words argument of pfz_lev_rows for a pattern of m code points."""
    if m <= 32:
        return 0
    for nw in (1, 2, 4, 8, 16):
        if m <= 64 * nw:
            return nw
    raise ValueError(f"from-string of {m} code points exceeds the supported maximum of {MAX_LEN}")


def _alphabet_batches(blob, offsets):
    """Split the from-rows into consecutive batches whose joint alphabet has <= 255 code points."""
    n = len(offsets) - 1
    if n == 0:
        return []
    if len(np.unique(blob)) <= 255:
        return [(0, n)]
    batches, lo, cur = [], 0, set()
    for i in range(n):
        cps = set(np.unique(blob[offsets[i]:offsets[i + 1]]).tolist())
        if len(cps) > 255:
            raise ValueError(f"from-string {i} has more than 255 distinct code points")
        if len(cur | cps) > 255:
            batches.append((lo, i)); lo, cur = i, set()
        cur |= cps
    batches.append((lo, n))
    return batches


def symbol_table(cps):
    """Code point -> byte symbol: the distinct code points cps (ascending) get 1, 2, ... and every other code point 0."""
    table = np.zeros(N_CODE_POINTS, dtype=np.uint8)
    ok = cps < N_CODE_POINTS
    table[cps[ok]] = np.arange(1, len(cps) + 1, dtype=np.uint8)[:int(ok.sum())]
    return table


def group_word_offsets(lens):
    """First 32-bit word of each group of 32 strings (lens in layout order) in the packed to-side layout, and the total at
    the end: a group holds ceil(its longest / 4) x 32 words."""
    n = len(lens)
    gmax = np.maximum.reduceat(lens, np.arange(0, n, 32)) if n else np.zeros(0, np.int64)
    goff = np.zeros((n + 31) // 32 + 1, dtype=np.int64)
    np.cumsum(((gmax + 3) // 4) * 32, out=goff[1:])
    return goff


def inverse_order(order):
    """pos_of[order[p]] = p: the sorted position of every to-index (the candidate kernels' pos_of)."""
    pos_of = np.empty(len(order), dtype=np.int32)
    pos_of[order] = np.arange(len(order), dtype=np.int32)
    return pos_of


def _blob_to_dev(b):
    if b.size == 0:
        return torch.zeros(1, dtype=torch.int32, device=_dev())
    return _to_dev(b).to(torch.int32) if b.dtype == np.uint8 else _to_dev(b.view(np.int32), torch.int32)


class EditQueries:
    """A from-list staged in HBM: UTF-32 blob + offsets, the rows of every word class, and per alphabet batch
    the code-point -> byte-symbol table (the kernel's symbols are bytes, see pfz.h)."""

    def __init__(self, from_list):
        self.n = len(from_list)
        blob, off, _ = pack_strings(from_list)
        lens = np.diff(off)
        if self.n and lens.max() > MAX_LEN:
            raise ValueError(f"from-string {int(lens.argmax())} has {int(lens.max())} code points; the edit-distance "
                             f"kernel supports at most {MAX_LEN}")
        self.lens = lens
        self.n_chars = int(blob.size)
        self.h2d_bytes = blob.nbytes + off.nbytes
        if self.n == 0:
            self.batches = []
            return
        self.d_blob = _blob_to_dev(blob)
        self.d_off = _to_dev(off)
        classes = np.select([lens <= 32, lens <= 64, lens <= 128, lens <= 256, lens <= 512], [0, 1, 2, 4, 8], 16).astype(np.int32)
        self.batches = []                                   # [(d_table, [(n_words, d_ids, n_ids), ...])]
        for lo, hi in _alphabet_batches(blob, off):
            table = symbol_table(np.unique(blob[off[lo]:off[hi]]).astype(np.int64))
            groups = []
            for nw in (0, 1, 2, 4, 8, 16):
                ids = np.nonzero(classes[lo:hi] == nw)[0].astype(np.int32) + lo
                if len(ids):
                    groups.append((nw, _to_dev(ids), len(ids)))
                    self.h2d_bytes += ids.nbytes
            self.batches.append((_to_dev(table), groups))
            self.h2d_bytes += table.nbytes


class EditTargets:
    """A to-list (or one row-block shard of it) staged in HBM: sorted by length, groups of 32, transposed,
    4 byte-symbols per 32-bit word (filled per alphabet batch by pfz_lev_pack)."""

    def __init__(self, to_list):
        self.n = len(to_list)
        blob, off, _ = pack_strings(to_list)
        self.n_chars = int(blob.size)
        self.h2d_bytes = blob.nbytes + off.nbytes
        if self.n == 0:
            return
        dev = _dev()
        self.d_blob = _blob_to_dev(blob)
        self.d_off = _to_dev(off)
        tlens = np.diff(off)
        self.lens = tlens
        order = np.argsort(tlens, kind="stable").astype(np.int32)
        self.n_grp = (self.n + 31) // 32
        goff = group_word_offsets(tlens[order])
        self.d_order = _to_dev(order); self.d_goff = _to_dev(goff)
        self.d_pos_of = _to_dev(inverse_order(order))        # candidate mode: to-index -> sorted position
        self.h2d_bytes += order.nbytes + goff.nbytes + order.nbytes
        self.packed = torch.empty(max(int(goff[-1]), 1), dtype=torch.int32, device=dev)
        self.slen = torch.empty(self.n, dtype=torch.int32, device=dev)


class KeptTargets:
    """The to-side a matcher staged last (EditTargets for K3, fuzzy.FuzzTargets for K3b), the device it lives on and a copy of
    the list it was staged from.  Neither depends on the from-list (the alphabet-dependent packing is redone per call), so a
    later call whose to-list is equal (same length, == element by element) can score against it without staging it again."""

    def __init__(self):
        self.clear()

    def clear(self):
        self.key = self.strings = self.staged = None

    def stage(self, kind, to_list, make, reuse):
        """The kept staging of `to_list` when `reuse` and it matches (kind, device, list); otherwise make(to_list), kept."""
        key = (kind, torch.cuda.current_device() if torch.cuda.is_available() else -1)
        if (reuse and self.staged is not None and self.key == key and len(self.strings) == len(to_list)
                and self.strings == list(to_list)):
            return self.staged
        self.clear()
        staged = make(to_list)
        self.key, self.strings, self.staged = key, list(to_list), staged
        return staged


def default_splits(n_from, n_grp):
    # ~4 (pattern, to-split) tasks per resident warp: patterns differ in length, finer tasks balance the tail
    want = 4 * 132 * 48
    return max(1, min(n_grp, (want + max(n_from, 1) - 1) // max(n_from, 1)))


def _word_classes(Q, T):
    """Per alphabet batch of Q: pack T under the batch's symbol table (pfz_lev_pack), then yield one
    (d_table, n_words, d_ids, n_ids) per word class of the batch."""
    for d_table, groups in Q.batches:
        _lib.call("pfz_lev_pack", _p(T.d_blob), _p(T.d_off), _p(T.d_order), T.n, _p(d_table), _p(T.d_goff), _p(T.packed), _p(T.slen),
                  _stream())
        for nw, d_ids, n_ids in groups:
            yield d_table, nw, d_ids, n_ids


def _gate_fill(metric, score_cutoff):
    """Gate of a row with fewer than k OSA candidates: the cutoff (norm_dl), or no bound (raw dl has no cutoff)."""
    return float(score_cutoff) if metric == "norm_dl" else float("-inf")


def _empty(n_from, k):
    """Rows with nothing to score: (idx, score, dist) [n_from] for the arg-best (k = 0), (idx, score) [n_from, k] for the k best;
    every slot empty (-1, 0.0, -1)."""
    dev = _dev()
    shape = (n_from, k) if k else (n_from,)
    out = (torch.full(shape, -1, dtype=torch.int32, device=dev), torch.zeros(shape, dtype=torch.float64, device=dev))
    return out if k else out + (torch.full(shape, -1, dtype=torch.int32, device=dev),)


def _rebase(idx, to_index_base):
    """to_index_base added to the found indices (row-block shards); empty slots stay -1."""
    return torch.where(idx >= 0, idx + int(to_index_base), idx) if to_index_base else idx


def _edit_rows(Q, T, metric, score_cutoff, exclude_self, self_shift, k, n_splits=None, cand=None, matrix=None, dl_gate=True,
               weights=None):
    """Score Q against T with pfz_lev_rows, every alphabet batch and word class, and return the rows' results: k = 0 the
    arg-best (idx, score, dist) [n_from], k >= 1 the k best (idx, score) [n_from, k].
    cand None: all pairs over n_splits to-splits (None: default_splits), merged by pfz_lev_merge (the arg-best, even with one
    split) or by pfz_topk_merge (the k best, more than one split).  cand (check_candidates): each row's own list, one split, no
    merge.  matrix (arg-best, int32 [>= n_from, >= n_to] or None) receives the distances.
    On all pairs a DL metric is gated per word class, unless dl_gate is False or a matrix is wanted: the same call with the
    OSA metric of DL_GATE, merged, gives each row's k-th best OSA score (k = 1 for the arg-best; _gate_fill when it has fewer).
    weights (check_weights, not None): weighted Levenshtein by pfz_wlev_rows instead; metric, matrix and dl_gate are unused."""
    n_from = Q.n
    if n_from == 0 or T.n == 0 or (cand is not None and cand.shape[1] == 0):
        return _empty(n_from, k)
    dev = _dev()
    if cand is not None:
        n_splits = 1
    elif n_splits is None:
        n_splits = default_splits(n_from, T.n_grp)
    n_splits = max(1, min(int(n_splits), T.n_grp))
    shape = (n_splits, n_from, k) if k else (n_splits, n_from)
    part = [torch.full(shape, -1, dtype=torch.int32, device=dev), torch.zeros(shape, dtype=torch.float64, device=dev)]
    if not k:
        part.append(torch.full(shape, -1, dtype=torch.int32, device=dev))
    counter = torch.zeros(n_splits, dtype=torch.int32, device=dev)
    src = (_p(cand), int(cand.shape[1]), _p(T.d_pos_of)) if cand is not None else (None, 0, None)

    def rows(d_table, nw, d_ids, n_ids, m, mat, gate):
        if weights is not None:
            _lib.call("pfz_wlev_rows", _p(Q.d_blob), _p(Q.d_off), n_from, _p(d_ids), n_ids, nw, _p(d_table), _p(T.packed), _p(T.d_goff),
                      _p(T.slen), _p(T.d_order), T.n, *weights, float(score_cutoff), int(bool(exclude_self)), int(self_shift), n_splits,
                      k, *src, _p(part[0]), _p(part[1]), _p(part[2] if not k else None), _p(counter), _stream())
            return
        _lib.call("pfz_lev_rows", _p(Q.d_blob), _p(Q.d_off), n_from, _p(d_ids), n_ids, nw, _p(d_table), _p(T.packed), _p(T.d_goff),
                  _p(T.slen), _p(T.d_order), T.n, METRIC[m], float(score_cutoff), int(bool(exclude_self)), int(self_shift), n_splits, k,
                  *src, _p(part[0]), _p(part[1]), _p(part[2] if not k else None), _p(mat), int(mat.stride(0)) if mat is not None else 0,
                  _p(gate), _p(counter), _stream())

    def merged():
        if cand is not None:
            return tuple(t[0] for t in part)
        if not k:
            return lev_merge(*part)
        return (part[0][0], part[1][0]) if n_splits == 1 else topk_merge(part[0], part[1], k)

    gated = metric in DL_GATE and cand is None and matrix is None and dl_gate
    for cls in _word_classes(Q, T):
        gate = None
        if gated:
            rows(*cls, DL_GATE[metric], None, None)
            gi, gs = merged()[:2]
            if k:
                gi, gs = gi[:, k - 1], gs[:, k - 1]
            gate = torch.where(gi >= 0, gs, _gate_fill(metric, score_cutoff)).contiguous()
        rows(*cls, metric, matrix, gate)
    return merged()


def edit_argbest_staged(Q, T, metric="ratio", score_cutoff=0.0, exclude_self=False, self_shift=0, want_matrix=False,
                        n_splits=None, to_index_base=0, dl_gate=True):
    """Kernels only.  Returns (best_idx int32[n_from] (-1 = none; + to_index_base otherwise), best_score float64[n_from],
    best_dist int32[n_from] [, matrix int32[n_from, n_to]]) as device tensors.
    dl / norm_dl: per word class an OSA arg-best pass and its split merge give each row's gate, then the DL pass;
    dl_gate=False (for timing) skips the OSA pass, and a matrix is computed without it."""
    if want_matrix and (metric in JARO_METRICS or metric in SEQ_METRICS):
        raise ValueError(f"want_matrix=True: the {metric!r} metric has no integer distance matrix")
    matrix = torch.zeros((max(Q.n, 1), max(T.n, 1)), dtype=torch.int32, device=_dev()) if want_matrix else None
    bi, bs, bd = _edit_rows(Q, T, metric, score_cutoff, exclude_self, self_shift, 0, n_splits, matrix=matrix, dl_gate=dl_gate)
    out = (_rebase(bi, to_index_base), bs, bd)
    return out + (matrix[:Q.n, :T.n],) if want_matrix else out


def _stage(from_list, to_list, kept, reuse):
    """EditQueries of from_list and EditTargets of to_list, the latter taken from kept (KeptTargets) when reuse allows it."""
    _dev()
    Q = EditQueries(from_list)
    T = kept.stage(("k3", 0), to_list, EditTargets, reuse) if kept is not None else EditTargets(to_list)
    return Q, T


def edit_argbest(from_list, to_list, metric="ratio", score_cutoff=0.0, exclude_self=False, self_shift=0,
                 want_matrix=False, n_splits=None, dl_gate=True, kept=None, reuse=False):
    """Host lists in, device tensors out (see edit_argbest_staged).  kept (KeptTargets): where the staged to-side is kept;
    reuse: take it from there when it was staged from an equal to_list."""
    Q, T = _stage(from_list, to_list, kept, reuse)
    return edit_argbest_staged(Q, T, metric, score_cutoff, exclude_self, self_shift, want_matrix, n_splits, dl_gate=dl_gate)


TOPK_MAX = 32
TOPK_METRICS = ("norm_lev", "ratio", "jaro", "jaro_winkler", "norm_osa", "norm_dl") + SEQ_METRICS


def check_top_n(k):
    """top_n of the edit-distance matchers: an int in 1..32 (the k best of a row are held in one warp's registers)."""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= TOPK_MAX:
        raise ValueError(f"top_n must be an int from 1 to {TOPK_MAX}, got {k!r}")
    return int(k)


def edit_topk_staged(Q, T, k, metric="ratio", score_cutoff=0.0, exclude_self=False, self_shift=0, n_splits=None, to_index_base=0,
                     dl_gate=True):
    """Kernels only: the k best to-strings per from-string (pfz_lev_rows, then pfz_topk_merge over the to-splits), with the
    candidates and the key of edit_argbest_staged.  Returns device (idx int32[n_from, k] (-1 = empty slot; + to_index_base
    otherwise), score float64[n_from, k] (0.0 in empty slots)).
    norm_dl: per word class a norm_osa top-k pass and its split merge give each row's gate (its k-th best OSA score), then
    the DL pass; dl_gate=False (for timing) skips the OSA pass."""
    k = check_top_n(k)
    if metric not in TOPK_METRICS:
        raise ValueError(f"top-k is available for the metrics {TOPK_METRICS}, not {metric!r}")
    idx, score = _edit_rows(Q, T, metric, score_cutoff, exclude_self, self_shift, k, n_splits, dl_gate=dl_gate)
    return _rebase(idx, to_index_base), score


def edit_topk(from_list, to_list, k, metric="ratio", score_cutoff=0.0, exclude_self=False, self_shift=0, n_splits=None, dl_gate=True,
              kept=None, reuse=False):
    """Host lists in, device tensors out (see edit_topk_staged); kept and reuse as in edit_argbest."""
    k = check_top_n(k)
    Q, T = _stage(from_list, to_list, kept, reuse)
    return edit_topk_staged(Q, T, k, metric, score_cutoff, exclude_self, self_shift, n_splits, dl_gate=dl_gate)


def lev_merge(part_idx, part_score, part_dist):
    """[n_lists, n_from] partial bests (GLOBAL indices) -> the canonical best per row (score desc, index asc)."""
    n_lists, n_from = part_idx.shape
    dev = part_idx.device
    bi = torch.full((max(n_from, 1),), -1, dtype=torch.int32, device=dev)
    bs = torch.zeros(max(n_from, 1), dtype=torch.float64, device=dev)
    bd = torch.full((max(n_from, 1),), -1, dtype=torch.int32, device=dev)
    _lib.call("pfz_lev_merge", _p(part_idx.contiguous()), _p(part_score.contiguous()), _p(part_dist.contiguous()), n_lists, n_from,
              _p(bi), _p(bs), _p(bd), _stream())
    return bi[:n_from], bs[:n_from], bd[:n_from]


def check_candidates(cand, n_from, n_to):
    """A candidate array for the cand kernels: a CUDA int32 tensor [n_from, c] (made contiguous) whose entries are to-indices
    in [0, n_to) or -1.  Indices must be distinct within a row (the top-k epilogue needs it; TF-IDF's rows are); that is not
    checked.  The range check costs one device-to-host read."""
    import torch as _t
    if not isinstance(cand, _t.Tensor) or cand.dtype != _t.int32 or cand.dim() != 2 or not cand.is_cuda:
        raise ValueError("candidates must be a CUDA int32 tensor [n_from, c]")
    if cand.shape[0] != n_from:
        raise ValueError(f"candidates have {cand.shape[0]} rows for {n_from} from-strings")
    cand = cand.contiguous()
    if cand.numel() and bool(((cand < -1) | (cand >= n_to)).any()):
        raise ValueError(f"candidate indices must lie in [-1, {n_to})")
    return cand


def edit_cand_topk_staged(Q, T, cand, k, metric="ratio", score_cutoff=0.0, exclude_self=False, self_shift=0):
    """Kernels only (pfz_lev_rows in candidate mode): per from-row the k best to-strings among its candidates cand[i]
    (check_candidates), under the metrics, cutoffs, self-exclusion and key of edit_argbest_staged / edit_topk_staged.
    k = 1 returns what edit_argbest_staged returns (best_idx, best_score, best_dist), any metric; k > 1 returns
    (idx int32[n_from, k], score float64[n_from, k]) as edit_topk_staged, metrics TOPK_METRICS.  A row with no candidate that
    passes gets (-1, 0.0).  dl / norm_dl run without the OSA gate (a row's list is short)."""
    k = check_top_n(k)
    if k > 1 and metric not in TOPK_METRICS:
        raise ValueError(f"top-k is available for the metrics {TOPK_METRICS}, not {metric!r}")
    if metric not in METRIC:
        raise ValueError(f"unknown metric {metric!r}")
    cand = check_candidates(cand, Q.n, T.n)
    # k = 1 takes the arg-best epilogue, which also gives the distance
    return _edit_rows(Q, T, metric, score_cutoff, exclude_self, self_shift, 0 if k == 1 else k, cand=cand)


def edit_cand_topk(from_list, to_list, cand, k, metric="ratio", score_cutoff=0.0, exclude_self=False, kept=None, reuse=False):
    """Host lists in, device tensors out (see edit_cand_topk_staged); kept and reuse as in edit_argbest."""
    k = check_top_n(k)
    Q, T = _stage(from_list, to_list, kept, reuse)
    return edit_cand_topk_staged(Q, T, cand, k, metric, score_cutoff, exclude_self)


# ---- weighted Levenshtein (DESIGN.md 4.17) ------------------------------------------------------------------------------------
WLEV_MAX_WEIGHT = 65535                 # PFZ_WLEV_MAX_WEIGHT


def check_weights(weights):
    """rapidfuzz's Levenshtein `weights` = (insertion, deletion, substitution): None (unit costs) or a tuple / list of three ints
    (Python or numpy integers, not bool), each in [0, WLEV_MAX_WEIGHT].  Returns None or a tuple of Python ints; anything else
    raises ValueError."""
    if weights is None:
        return None
    if (not isinstance(weights, (tuple, list)) or len(weights) != 3
            or not all(isinstance(w, (int, np.integer)) and not isinstance(w, bool) and 0 <= w <= WLEV_MAX_WEIGHT for w in weights)):
        raise ValueError(f"weights must be None or three ints (insertion, deletion, substitution) in [0, {WLEV_MAX_WEIGHT}], "
                         f"got {weights!r}")
    return tuple(int(w) for w in weights)


def uniform_weight(weights):
    """w for weights (w, w, w) with w >= 1, and 1 for None: D = w * lev and M = w * max(|a|, |b|), so the scores are norm_lev's
    bit for bit.  0 for every other triple."""
    if weights is None:
        return 1
    wi, wd, ws = weights
    return wi if wi == wd == ws and wi >= 1 else 0


def _wlev_rows(Q, T, weights, score_cutoff, exclude_self, self_shift, k, n_splits=None, cand=None):
    """_edit_rows for weighted Levenshtein: uniform weights take the norm_lev path (its arg-best distances times w, saturated at
    2^31 - 1 as pfz_wlev_rows saturates D), any other triple pfz_wlev_rows."""
    weights = check_weights(weights)
    w = uniform_weight(weights)
    if not w:
        return _edit_rows(Q, T, None, score_cutoff, exclude_self, self_shift, k, n_splits, cand, weights=weights)
    out = _edit_rows(Q, T, "norm_lev", score_cutoff, exclude_self, self_shift, k, n_splits, cand)
    if k or w == 1:
        return out
    d = (out[2].to(torch.int64) * w).clamp(max=2**31 - 1).to(torch.int32)
    return out[:2] + (torch.where(out[2] >= 0, d, out[2]),)


def edit_wlev_argbest_staged(Q, T, weights, score_cutoff=0.0, exclude_self=False, self_shift=0, want_matrix=False, n_splits=None,
                             to_index_base=0):
    """Kernels only: per from-string the best to-string under rapidfuzz's Levenshtein.normalized_similarity(from, to,
    weights=weights) (score 1 - D/M, key and cutoff as norm_lev).  Returns device (best_idx int32[n_from] (-1 = none;
    + to_index_base otherwise), best_score float64[n_from], best_dist int32[n_from] = the weighted distance D, saturated at
    2^31 - 1).  There is no distance matrix: want_matrix=True raises ValueError."""
    if want_matrix:
        raise ValueError("want_matrix=True: weighted Levenshtein has no distance matrix")
    bi, bs, bd = _wlev_rows(Q, T, weights, score_cutoff, exclude_self, self_shift, 0, n_splits)
    return _rebase(bi, to_index_base), bs, bd


def edit_wlev_argbest(from_list, to_list, weights, score_cutoff=0.0, exclude_self=False, self_shift=0, want_matrix=False,
                      n_splits=None, kept=None, reuse=False):
    """Host lists in, device tensors out (see edit_wlev_argbest_staged); kept and reuse as in edit_argbest."""
    check_weights(weights)
    Q, T = _stage(from_list, to_list, kept, reuse)
    return edit_wlev_argbest_staged(Q, T, weights, score_cutoff, exclude_self, self_shift, want_matrix, n_splits)


def edit_wlev_topk_staged(Q, T, k, weights, score_cutoff=0.0, exclude_self=False, self_shift=0, n_splits=None, to_index_base=0):
    """Kernels only: the k best to-strings per from-string under weighted Levenshtein, with the candidates and key of
    edit_wlev_argbest_staged.  Returns device (idx int32[n_from, k] (-1 = empty slot; + to_index_base otherwise),
    score float64[n_from, k] (0.0 in empty slots))."""
    k = check_top_n(k)
    idx, score = _wlev_rows(Q, T, weights, score_cutoff, exclude_self, self_shift, k, n_splits)
    return _rebase(idx, to_index_base), score


def edit_wlev_topk(from_list, to_list, k, weights, score_cutoff=0.0, exclude_self=False, self_shift=0, n_splits=None, kept=None,
                   reuse=False):
    """Host lists in, device tensors out (see edit_wlev_topk_staged); kept and reuse as in edit_argbest."""
    k = check_top_n(k)
    check_weights(weights)
    Q, T = _stage(from_list, to_list, kept, reuse)
    return edit_wlev_topk_staged(Q, T, k, weights, score_cutoff, exclude_self, self_shift, n_splits)


def edit_wlev_cand_topk_staged(Q, T, cand, k, weights, score_cutoff=0.0, exclude_self=False, self_shift=0):
    """Kernels only (pfz_wlev_rows in candidate mode): per from-row the k best to-strings among its candidates cand[i]
    (check_candidates) under weighted Levenshtein.  k = 1 returns what edit_wlev_argbest_staged returns, k > 1 what
    edit_wlev_topk_staged returns."""
    k = check_top_n(k)
    cand = check_candidates(cand, Q.n, T.n)
    return _wlev_rows(Q, T, weights, score_cutoff, exclude_self, self_shift, 0 if k == 1 else k, cand=cand)


def edit_wlev_cand_topk(from_list, to_list, cand, k, weights, score_cutoff=0.0, exclude_self=False, kept=None, reuse=False):
    """Host lists in, device tensors out (see edit_wlev_cand_topk_staged); kept and reuse as in edit_argbest."""
    k = check_top_n(k)
    check_weights(weights)
    Q, T = _stage(from_list, to_list, kept, reuse)
    return edit_wlev_cand_topk_staged(Q, T, cand, k, weights, score_cutoff, exclude_self)
