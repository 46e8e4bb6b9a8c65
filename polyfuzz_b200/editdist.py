"""K3 host driver: all-pairs edit distance with per-row arg-best on the GPU (include/pfz.h, pfz_lev_*).

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
                again, so dl("CA", "ABC") = 2); computed by pfz_dl_*, gated by an OSA pass (DESIGN.md 4.10)
The Jaro metrics are computed on code points, from-string first (the reference calls scorer(from_string, to_string),
polyfuzz/models/_distance.py:98); their best_dist is the number of matching characters, and they have no distance
matrix (want_matrix=True raises ValueError).
Best match of a from-string = first to-string (lowest index) with the maximal score >= score_cutoff; the top-k functions
return the k best under the same key (score desc, index asc), k <= 32.

Two levels: `EditQueries` / `EditTargets` stage a from-list / to-list in HBM once (host packing, length sort,
alphabet batches); `edit_argbest_staged` only enqueues kernels, so a staged pair can be scored repeatedly
(bench.py's device-timed leg, the multi-GPU shards) without touching the host lists again.  `KeptTargets` holds a
matcher's last staged to-side, which a `re_train=False` call with an equal to-list scores against again.
"""
import numpy as np
import torch

from . import _lib
from .engine import _dev, _p, _stream, _to_dev, topk_merge
from .strings import pack_strings

METRIC = {"lev": 0, "indel": 1, "norm_lev": 2, "ratio": 3, "jaro": 4, "jaro_winkler": 5, "osa": 6, "norm_osa": 7, "dl": 8,
          "norm_dl": 9}
JARO_METRICS = ("jaro", "jaro_winkler")
# DL metric -> the OSA metric whose k-th best score gates it (norm_osa <= norm_dl pair by pair, DESIGN.md 4.10)
DL_GATE = {"dl": "osa", "norm_dl": "norm_osa"}
N_CODE_POINTS = 0x110000
MAX_LEN = 1024


def _word_class(m):
    """n_words argument of pfz_lev_argbest for a pattern of m code points."""
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
        self.h2d_bytes += order.nbytes + goff.nbytes
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


def _k3_head(Q, T, cls, metric, score_cutoff, exclude_self, self_shift, n_splits):
    """The leading arguments of pfz_lev_argbest, pfz_lev_topk, pfz_dl_argbest and pfz_dl_topk (from_blob .. n_splits)."""
    d_table, nw, d_ids, n_ids = cls
    return (_p(Q.d_blob), _p(Q.d_off), Q.n, _p(d_ids), n_ids, nw, _p(d_table), _p(T.packed), _p(T.d_goff), _p(T.slen),
            _p(T.d_order), T.n, METRIC[metric], float(score_cutoff), int(bool(exclude_self)), int(self_shift), n_splits)


def _gate_fill(metric, score_cutoff):
    """Gate of a row with fewer than k OSA candidates: the cutoff (norm_dl), or no bound (raw dl has no cutoff)."""
    return float(score_cutoff) if metric == "norm_dl" else float("-inf")


def edit_argbest_staged(Q, T, metric="ratio", score_cutoff=0.0, exclude_self=False, self_shift=0, want_matrix=False,
                        n_splits=None, to_index_base=0, dl_gate=True):
    """Kernels only.  Returns (best_idx int32[n_from] (-1 = none; + to_index_base otherwise), best_score float64[n_from],
    best_dist int32[n_from] [, matrix int32[n_from, n_to]]) as device tensors.
    dl / norm_dl: per word class an OSA arg-best pass and its split merge give each row's gate, then pfz_dl_argbest;
    dl_gate=False (for timing) skips the OSA pass, and a matrix is computed without it."""
    if want_matrix and metric in JARO_METRICS:
        raise ValueError(f"want_matrix=True: the {metric!r} metric has no integer distance matrix")
    dev = _dev()
    n_from, n_to = Q.n, T.n
    best_idx = torch.full((max(n_from, 1),), -1, dtype=torch.int32, device=dev)
    best_score = torch.zeros(max(n_from, 1), dtype=torch.float64, device=dev)
    best_dist = torch.full((max(n_from, 1),), -1, dtype=torch.int32, device=dev)
    matrix = torch.zeros((max(n_from, 1), max(n_to, 1)), dtype=torch.int32, device=dev) if want_matrix else None
    if n_from == 0 or n_to == 0:
        out = (best_idx[:n_from], best_score[:n_from], best_dist[:n_from])
        return out + (matrix[:n_from, :n_to],) if want_matrix else out
    if n_splits is None:
        n_splits = default_splits(n_from, T.n_grp)
    n_splits = max(1, min(int(n_splits), T.n_grp))
    part_idx = torch.full((n_splits, n_from), -1, dtype=torch.int32, device=dev)
    part_score = torch.zeros((n_splits, n_from), dtype=torch.float64, device=dev)
    part_dist = torch.full((n_splits, n_from), -1, dtype=torch.int32, device=dev)
    counter = torch.zeros(n_splits, dtype=torch.int32, device=dev)
    mat = (_p(matrix), int(matrix.stride(0)) if matrix is not None else 0)
    for cls in _word_classes(Q, T):
        head = lambda m: _k3_head(Q, T, cls, m, score_cutoff, exclude_self, self_shift, n_splits)  # noqa: E731
        if metric not in DL_GATE:
            _lib.call("pfz_lev_argbest", *head(metric), _p(part_idx), _p(part_score), _p(part_dist), *mat, _p(counter), _stream())
            continue
        gate = None
        if dl_gate and not want_matrix:
            _lib.call("pfz_lev_argbest", *head(DL_GATE[metric]), _p(part_idx), _p(part_score), _p(part_dist), None, 0, _p(counter),
                      _stream())
            _lib.call("pfz_lev_merge", _p(part_idx), _p(part_score), _p(part_dist), n_splits, n_from, _p(best_idx),
                      _p(best_score), _p(best_dist), _stream())
            gate = torch.where(best_idx >= 0, best_score, _gate_fill(metric, score_cutoff))
        _lib.call("pfz_dl_argbest", *head(metric), _p(part_idx), _p(part_score), _p(part_dist), *mat, _p(gate), _p(counter),
                  _stream())
    _lib.call("pfz_lev_merge", _p(part_idx), _p(part_score), _p(part_dist), n_splits, n_from, _p(best_idx), _p(best_score),
              _p(best_dist), _stream())
    if to_index_base:
        best_idx = torch.where(best_idx >= 0, best_idx + int(to_index_base), best_idx)
    out = (best_idx[:n_from], best_score[:n_from], best_dist[:n_from])
    return out + (matrix[:n_from, :n_to],) if want_matrix else out


def edit_argbest(from_list, to_list, metric="ratio", score_cutoff=0.0, exclude_self=False, self_shift=0,
                 want_matrix=False, n_splits=None, dl_gate=True, kept=None, reuse=False):
    """Host lists in, device tensors out (see edit_argbest_staged).  kept (KeptTargets): where the staged to-side is kept;
    reuse: take it from there when it was staged from an equal to_list."""
    _dev()
    Q = EditQueries(from_list)
    T = kept.stage(("k3", 0), to_list, EditTargets, reuse) if kept is not None else EditTargets(to_list)
    return edit_argbest_staged(Q, T, metric, score_cutoff, exclude_self, self_shift, want_matrix, n_splits, dl_gate=dl_gate)


TOPK_MAX = 32
TOPK_METRICS = ("norm_lev", "ratio", "jaro", "jaro_winkler", "norm_osa", "norm_dl")


def check_top_n(k):
    """top_n of the edit-distance matchers: an int in 1..32 (the k best of a row are held in one warp's registers)."""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= TOPK_MAX:
        raise ValueError(f"top_n must be an int from 1 to {TOPK_MAX}, got {k!r}")
    return int(k)


def edit_topk_staged(Q, T, k, metric="ratio", score_cutoff=0.0, exclude_self=False, self_shift=0, n_splits=None, to_index_base=0,
                     dl_gate=True):
    """Kernels only: the k best to-strings per from-string (pfz_lev_topk, then pfz_topk_merge over the to-splits), with the
    candidates and the key of edit_argbest_staged.  Returns device (idx int32[n_from, k] (-1 = empty slot; + to_index_base
    otherwise), score float64[n_from, k] (0.0 in empty slots)).
    norm_dl: per word class a norm_osa top-k pass and its split merge give each row's gate (its k-th best OSA score), then
    pfz_dl_topk; dl_gate=False (for timing) skips the OSA pass."""
    k = check_top_n(k)
    if metric not in TOPK_METRICS:
        raise ValueError(f"top-k is available for the metrics {TOPK_METRICS}, not {metric!r}")
    dev = _dev()
    n_from, n_to = Q.n, T.n
    if n_from == 0 or n_to == 0:
        return (torch.full((n_from, k), -1, dtype=torch.int32, device=dev), torch.zeros((n_from, k), dtype=torch.float64, device=dev))
    if n_splits is None:
        n_splits = default_splits(n_from, T.n_grp)
    n_splits = max(1, min(int(n_splits), T.n_grp))
    part_idx = torch.full((n_splits, n_from, k), -1, dtype=torch.int32, device=dev)
    part_score = torch.zeros((n_splits, n_from, k), dtype=torch.float64, device=dev)
    counter = torch.zeros(n_splits, dtype=torch.int32, device=dev)
    for cls in _word_classes(Q, T):
        head = lambda m: _k3_head(Q, T, cls, m, score_cutoff, exclude_self, self_shift, n_splits)  # noqa: E731
        if metric not in DL_GATE:
            _lib.call("pfz_lev_topk", *head(metric), k, _p(part_idx), _p(part_score), _p(counter), _stream())
            continue
        gate = None
        if dl_gate:
            _lib.call("pfz_lev_topk", *head(DL_GATE[metric]), k, _p(part_idx), _p(part_score), _p(counter), _stream())
            gi, gs = (part_idx[0], part_score[0]) if n_splits == 1 else topk_merge(part_idx, part_score, k)
            gate = torch.where(gi[:, k - 1] >= 0, gs[:, k - 1], _gate_fill(metric, score_cutoff)).contiguous()
        _lib.call("pfz_dl_topk", *head(metric), k, _p(part_idx), _p(part_score), _p(gate), _p(counter), _stream())
    idx, score = (part_idx[0], part_score[0]) if n_splits == 1 else topk_merge(part_idx, part_score, k)
    if to_index_base:
        idx = torch.where(idx >= 0, idx + int(to_index_base), idx)
    return idx, score


def edit_topk(from_list, to_list, k, metric="ratio", score_cutoff=0.0, exclude_self=False, self_shift=0, n_splits=None, dl_gate=True,
              kept=None, reuse=False):
    """Host lists in, device tensors out (see edit_topk_staged); kept and reuse as in edit_argbest."""
    k = check_top_n(k)
    _dev()
    Q = EditQueries(from_list)
    T = kept.stage(("k3", 0), to_list, EditTargets, reuse) if kept is not None else EditTargets(to_list)
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
