"""K3b host driver: rapidfuzz's token / partial / weighted scorers (WRatio, partial_ratio, token_sort_ratio, token_set_ratio,
token_ratio, partial_token_*_ratio, QRatio) over the |from| x |to| grid with a fused per-row arg-best on the GPU
(include/pfz.h, pfz_fuzz_rows; csrc/pfz_fuzz.cu).

Replaces the scorer loop of polyfuzz/models/_rapidfuzz.py:99-113 (process.extractOne with scorer=fuzz.WRatio, the
reference's default, :48) and polyfuzz/models/_distance.py:89-102 for those scorers.  The host only packs each list into a
UTF-32 blob and uploads it; the token tables are built on the device (pfz_tok_*, csrc/pfz_tok.cu): per string the
whitespace tokens (str.split(), as rapidfuzz), the derived strings S(s) = sorted tokens joined and U(s) = distinct sorted
tokens joined, the sorted distinct token ids over one dictionary numbered in sorted token order, and a 64-bit Bloom
signature of the ids; every score is computed on the device.

A to-list is staged once into a `FuzzTargets` (its token tables, length order and pack buffers), which depends on no
from-list: a matcher keeps it across calls (editdist.KeptTargets), and each call only tokenises the from-list, joins the two
vocabularies and renumbers the kept to-side ids to the union (pfz_tok_union, pfz_tok_remap).

`fuzz_cand_topk` scores each from-row against its own candidate list only (editdist.check_candidates; DESIGN.md 4.16).
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .editdist import (_alphabet_batches, _blob_to_dev, _empty, _rebase, check_candidates, check_top_n, default_splits,
                       group_word_offsets, inverse_order, lev_merge, symbol_table)
from .engine import _dev, _p, _stream, _to_dev, topk_merge
from .strings import pack_strings

SCORER = {"ratio": 0, "QRatio": 1, "partial_ratio": 2, "token_sort_ratio": 3, "token_set_ratio": 4, "token_ratio": 5,
          "partial_token_sort_ratio": 6, "partial_token_set_ratio": 7, "partial_token_ratio": 8, "WRatio": 9}
MAX_LEN = 1024                                             # code points per from-string (every variant); to-strings: any length


def word_class(lens):
    """64-bit words per from-string mask for the longest of its variants: <= 64 -> 1, <= 128 -> 2, <= 256 -> 4, <= 512 -> 8,
    else 16 (the 8- and 16-word classes run one CTA per from-row)."""
    return np.select([lens <= 64, lens <= 128, lens <= 256, lens <= 512], [1, 2, 4, 8], 16).astype(np.int32)


class TokSide:
    """One string list tokenised on the device (pfz_tok_side): the s, S(s), U(s) blobs + offsets, the list's own sorted
    vocabulary, each string's distinct token ids in that vocabulary (tok_ptr, tok_ids) and its token count.  The ids the
    kernels take are those of the union with the other list of the call (see _call_ids)."""

    def __init__(self, strings):
        dev = _dev()
        self.n = len(strings)
        blob, off, _ = pack_strings(strings)
        self.host = (blob, off)
        self.lens = np.diff(off)
        n_chars = int(off[-1]) if len(off) else 0
        cap = max(n_chars, 1)
        self.d_blob, self.d_off = _blob_to_dev(blob), _to_dev(off)
        self.d_n_all = torch.zeros(max(self.n, 1), dtype=torch.int32, device=dev)
        self.d_vocab_blob = torch.empty(cap, dtype=torch.int32, device=dev)
        self.d_vocab_off = torch.zeros(cap + 1, dtype=torch.int64, device=dev)
        self.d_tok_ptr = torch.zeros(self.n + 1, dtype=torch.int32, device=dev)
        self.d_tok_ids = torch.empty(cap, dtype=torch.int32, device=dev)
        self.d_S = (torch.empty(cap, dtype=torch.int32, device=dev), torch.zeros(self.n + 1, dtype=torch.int64, device=dev))
        self.d_U = (torch.empty(cap, dtype=torch.int32, device=dev), torch.zeros(self.n + 1, dtype=torch.int64, device=dev))
        counts = np.zeros(6, dtype=np.int64)
        _lib.call("pfz_tok_side", _p(self.d_blob), _p(self.d_off), self.n, n_chars, _p(self.d_n_all), _p(self.d_vocab_blob),
                  _p(self.d_vocab_off), _p(self.d_tok_ptr), _p(self.d_tok_ids), _p(self.d_S[1]), _p(self.d_S[0]), _p(self.d_U[1]),
                  _p(self.d_U[0]), ctypes.c_void_p(counts.ctypes.data), _stream())
        self.n_tokens, self.n_vocab, self.vocab_chars, _, _, self.n_ids = (int(x) for x in counts)

    def variant_lens(self):
        """|s|, |S(s)|, |U(s)| per string (host; one small D2H of the S and U offsets)."""
        return [self.lens, np.diff(self.d_S[1].cpu().numpy()), np.diff(self.d_U[1].cpu().numpy())]

    def ptrs(self, ids, sig):
        return [self.d_blob, self.d_off, self.d_S[0], self.d_S[1], self.d_U[0], self.d_U[1], self.d_tok_ptr, ids, sig, self.d_n_all]


class FuzzTargets:
    """A to-list (or one row-block shard of it) staged for K3b: its TokSide, ONE length order (by len(b)) for the three variants
    and each variant's group offsets and pack buffers (filled per alphabet batch by pfz_lev_pack).  Nothing in it depends on
    the from-list, so it can serve any number of calls."""

    def __init__(self, to_list):
        self.n = len(to_list)
        if self.n == 0:
            return
        dev = _dev()
        self.side = TokSide(to_list)
        lens = self.side.variant_lens()
        order = np.argsort(lens[0], kind="stable").astype(np.int32)
        self.n_grp = (self.n + 31) // 32
        self.d_order = _to_dev(order)
        self.d_pos_of = _to_dev(inverse_order(order))        # candidate mode: to-index -> sorted position
        self.packs = []
        for v in range(3):
            goff = group_word_offsets(lens[v][order])
            self.packs.append((torch.empty(max(int(goff[-1]), 1), dtype=torch.int32, device=dev), _to_dev(goff),
                               torch.empty(self.n, dtype=torch.int32, device=dev)))


def _call_ids(F, T, same):
    """The ids of one call: both sides renumbered to the union of their vocabularies (a monotone map, so each string's ids stay
    ascending), their signatures, and the union vocabulary (tok_blob, tok_off).  Returns (f_ids, f_sig, t_ids, t_sig, tok_blob,
    tok_off); a self-match (same) shares one side and its own vocabulary."""
    dev = _dev()

    def remap(S, d_map):
        ids = torch.empty(max(S.n_ids, 1), dtype=torch.int32, device=dev)
        sig = torch.empty(max(S.n, 1), dtype=torch.int64, device=dev)
        _lib.call("pfz_tok_remap", _p(S.d_tok_ptr), _p(S.d_tok_ids), S.n, _p(d_map), _p(ids), _p(sig), _stream())
        return ids, sig

    if same:
        ids, sig = remap(F, None)
        return ids, sig, ids, sig, F.d_vocab_blob, F.d_vocab_off
    map_f = torch.empty(max(F.n_vocab, 1), dtype=torch.int32, device=dev)
    map_t = torch.empty(max(T.n_vocab, 1), dtype=torch.int32, device=dev)
    u_blob = torch.empty(max(F.vocab_chars + T.vocab_chars, 1), dtype=torch.int32, device=dev)
    u_off = torch.zeros(F.n_vocab + T.n_vocab + 1, dtype=torch.int64, device=dev)
    n_u = torch.zeros(1, dtype=torch.int32, device=dev)
    _lib.call("pfz_tok_union", _p(F.d_vocab_blob), _p(F.d_vocab_off), F.n_vocab, _p(T.d_vocab_blob), _p(T.d_vocab_off), T.n_vocab,
              _p(map_f), _p(map_t), _p(u_blob), _p(u_off), _p(n_u), _stream())
    return remap(F, map_f) + remap(T, map_t) + (u_blob, u_off)


def _enqueue(from_list, to_list, scorer, score_cutoff, exclude_self, n_splits, self_shift, to_index_base, k, kept=None, reuse=False,
             cand=None):
    """Stage the from-list (and the to-list, unless `kept` -- an editdist.KeptTargets -- holds it already and `reuse` allows
    it), join the two vocabularies, and enqueue pfz_fuzz_rows for every alphabet batch and word class: the arg-best with part_*
    [n_splits, n_from] when k is None, else the k best with part_* [n_splits, n_from, k].  cand (a checked candidate array):
    each row's own list, one split.  Returns (part_idx, part_score, n_splits, staged):
    `staged` keeps the staged buffers alive until the caller has synchronised."""
    dev = _dev()
    n_from, n_to = len(from_list), len(to_list)
    same = to_list is from_list and not to_index_base
    if kept is not None:
        targets = kept.stage(("k3b", int(to_index_base)), to_list, FuzzTargets, reuse)
    else:
        targets = FuzzTargets(to_list)
    T = targets.side
    F = T if same else TokSide(from_list)
    # max(|s|, |S(s)|, |U(s)|) is |s|: S(s) keeps the tokens of s and at most as many separators
    fl = F.lens
    if len(fl) and fl.max() > MAX_LEN:
        raise ValueError(f"from-string {int(fl.argmax())} has {int(fl.max())} code points; the token / partial scorers "
                         f"support at most {MAX_LEN}")
    f_ids, f_sig, t_ids, t_sig, d_tok_blob, d_tok_off = _call_ids(F, T, same)
    d_order, packs = targets.d_order, targets.packs
    if cand is not None:
        n_splits = 1
    elif n_splits is None:
        n_splits = default_splits(n_from, targets.n_grp)
    n_splits = max(1, min(int(n_splits), targets.n_grp))
    shape = (n_splits, n_from) if k is None else (n_splits, n_from, k)
    part_idx = torch.full(shape, -1, dtype=torch.int32, device=dev)
    part_score = torch.zeros(shape, dtype=torch.float64, device=dev)
    counter = torch.zeros(n_splits, dtype=torch.int32, device=dev)
    classes = word_class(fl)
    fblob, foff = F.host
    keep = [f_ids, f_sig, t_ids, t_sig]
    for lo, hi in _alphabet_batches(fblob, foff):
        cps = np.unique(np.concatenate([fblob[foff[lo]:foff[hi]].astype(np.int64), np.array([0x20], dtype=np.int64)]))
        if len(cps) > 255:
            raise ValueError("a batch of from-strings has more than 254 distinct code points besides the space")
        d_table = _to_dev(symbol_table(cps)); keep.append(d_table)
        for v, (d_blob, d_off) in enumerate(((T.d_blob, T.d_off), T.d_S, T.d_U)):
            _lib.call("pfz_lev_pack", _p(d_blob), _p(d_off), _p(d_order), n_to, _p(d_table), _p(packs[v][1]), _p(packs[v][0]),
                      _p(packs[v][2]), _stream())
        for nw in (1, 2, 4, 8, 16):
            ids = np.nonzero(classes[lo:hi] == nw)[0].astype(np.int32) + lo
            if len(ids) == 0:
                continue
            d_ids = _to_dev(ids); keep.append(d_ids)
            tens = F.ptrs(f_ids, f_sig) + T.ptrs(t_ids, t_sig) + [d_ids, d_table]
            for v in range(3):
                tens += [packs[v][0], packs[v][1], packs[v][2]]
            tens += [d_order, d_tok_blob, d_tok_off, part_idx, part_score, counter, None]
            arr = (ctypes.c_void_p * len(tens))(*[t.data_ptr() if t is not None else 0 for t in tens])
            src = (_p(cand), int(cand.shape[1]), _p(targets.d_pos_of)) if cand is not None else (None, 0, None)
            _lib.call("pfz_fuzz_rows", arr, len(tens), n_from, len(ids), int(nw), n_to, SCORER[scorer], float(score_cutoff),
                      int(bool(exclude_self)), int(self_shift), n_splits, int(k or 0), *src, _stream())
    return part_idx, part_score, n_splits, (F, targets, keep, d_tok_blob, d_tok_off)


def _scores(from_list, to_list, scorer, score_cutoff, exclude_self, n_splits, self_shift, to_index_base, k, kept, reuse, cand=None):
    """The rows' results of the public functions: (idx, score) [n_from] for the arg-best (k None), [n_from, k] for the k best.
    _enqueue, then the split merge (pfz_lev_merge for the arg-best even with one split, pfz_topk_merge over more than one split,
    none in candidate mode), the synchronise and to_index_base added to the found indices."""
    if scorer not in SCORER:
        raise NotImplementedError(f"scorer {scorer!r} has no GPU implementation (supported: {sorted(SCORER)})")
    n_from, n_to = len(from_list), len(to_list)
    if cand is not None:
        cand = check_candidates(cand, n_from, n_to)
    if n_from == 0 or n_to == 0 or (cand is not None and cand.shape[1] == 0):
        return _empty(n_from, k or 0)[:2]
    part_idx, part_score, n_splits, staged = _enqueue(from_list, to_list, scorer, score_cutoff, exclude_self, n_splits, self_shift,
                                                      to_index_base, k, kept, reuse, cand)
    if cand is not None or (k is not None and n_splits == 1):
        idx, score = part_idx[0], part_score[0]
    elif k is None:
        idx, score, _ = lev_merge(part_idx, part_score, torch.full_like(part_idx, -1))
    else:
        idx, score = topk_merge(part_idx, part_score, k)
    torch.cuda.current_stream().synchronize()                  # the staged host buffers above go out of scope with this call
    return _rebase(idx, to_index_base), score


def fuzz_argbest(from_list, to_list, scorer="WRatio", score_cutoff=0.0, exclude_self=False, n_splits=None, self_shift=0,
                 to_index_base=0, kept=None, reuse=False):
    """Best to-string per from-string under a rapidfuzz scorer (scores in [0, 100]).  Returns device tensors
    (best_idx int32[n_from] (-1: no to-string reached score_cutoff), best_score float64[n_from]).
    exclude_self skips to-row == from-row + self_shift; to_index_base is added to the returned indices (row-block shards).
    kept (editdist.KeptTargets): where the staged to-side is kept; reuse: take it from there when it was staged from an equal
    to_list."""
    return _scores(from_list, to_list, scorer, score_cutoff, exclude_self, n_splits, self_shift, to_index_base, None, kept, reuse)


def fuzz_topk(from_list, to_list, k, scorer="WRatio", score_cutoff=0.0, exclude_self=False, n_splits=None, self_shift=0,
              to_index_base=0, kept=None, reuse=False):
    """The k best to-strings per from-string (1 <= k <= 32) under the candidates and key of fuzz_argbest (score desc, index asc).
    Returns device tensors (idx int32[n_from, k] (-1: empty slot), score float64[n_from, k] (0.0 in empty slots));
    exclude_self, self_shift, to_index_base, kept and reuse as in fuzz_argbest."""
    k = check_top_n(k)
    return _scores(from_list, to_list, scorer, score_cutoff, exclude_self, n_splits, self_shift, to_index_base, k, kept, reuse)


def fuzz_cand_topk(from_list, to_list, cand, k, scorer="WRatio", score_cutoff=0.0, exclude_self=False, kept=None, reuse=False):
    """The k best to-strings per from-string among its candidates cand[i] (editdist.check_candidates: device int32
    [n_from, c], -1 = empty slot), under the scores, cutoff and key of fuzz_argbest / fuzz_topk.  k = 1 returns what
    fuzz_argbest returns (best_idx int32[n_from], best_score float64[n_from]); k > 1 what fuzz_topk returns.  A row with no
    candidate that passes gets (-1, 0.0); exclude_self, kept and reuse as in fuzz_argbest."""
    k = check_top_n(k)
    return _scores(from_list, to_list, scorer, score_cutoff, exclude_self, 1, 0, 0, None if k == 1 else k, kept, reuse, cand)
