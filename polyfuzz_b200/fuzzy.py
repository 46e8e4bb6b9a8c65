"""K3b host driver: rapidfuzz's token / partial / weighted scorers (WRatio, partial_ratio, token_sort_ratio, token_set_ratio,
token_ratio, partial_token_*_ratio, QRatio) over the |from| x |to| grid with a fused per-row arg-best on the GPU
(include/pfz.h, pfz_fuzz_argbest; csrc/pfz_fuzz.cu).

Replaces the scorer loop of polyfuzz/models/_rapidfuzz.py:99-113 (process.extractOne with scorer=fuzz.WRatio, the
reference's default, :48) and polyfuzz/models/_distance.py:89-102 for those scorers.  The host side only marshals: per
string the whitespace tokens (str.split(), as rapidfuzz), the derived strings S(s) = sorted tokens joined and U(s) =
distinct sorted tokens joined, the sorted distinct token ids over one dictionary numbered in sorted token order, and a
64-bit Bloom signature of the ids; every score is computed on the device.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .editdist import _alphabet_batches, _blob_to_dev, check_top_n, default_splits, group_word_offsets, symbol_table
from .engine import _dev, _p, _stream, _to_dev, topk_merge
from .strings import pack_strings

SCORER = {"ratio": 0, "QRatio": 1, "partial_ratio": 2, "token_sort_ratio": 3, "token_set_ratio": 4, "token_ratio": 5,
          "partial_token_sort_ratio": 6, "partial_token_set_ratio": 7, "partial_token_ratio": 8, "WRatio": 9}
MAX_LEN = 1024                                             # code points per from-string (every variant); to-strings: any length


def word_class(lens):
    """64-bit words per from-string mask for the longest of its variants: <= 64 -> 1, <= 128 -> 2, <= 256 -> 4, <= 512 -> 8,
    else 16 (the 8- and 16-word classes run one CTA per from-row)."""
    return np.select([lens <= 64, lens <= 128, lens <= 256, lens <= 512], [1, 2, 4, 8], 16).astype(np.int32)


def _derive(strings):
    toks = [s.split() for s in strings]
    return toks, [" ".join(sorted(t)) for t in toks], [" ".join(sorted(set(t))) for t in toks]


class _Side:
    """One string list staged for the kernel: s, S(s), U(s) blobs + offsets, distinct token ids, signatures."""

    def __init__(self, strings, toks, sorted_joined, uniq_joined, tok_id):
        self.n = len(strings)
        self.host = []
        self.dev = []
        for lst in (strings, sorted_joined, uniq_joined):
            blob, off, _ = pack_strings(lst)
            self.host.append((blob, off))
            self.dev.append((_blob_to_dev(blob), _to_dev(off)))
        self.lens = [np.diff(off) for _, off in self.host]
        ptr = np.zeros(self.n + 1, dtype=np.int32)
        ids, sig = [], np.zeros(self.n, dtype=np.uint64)
        n_all = np.zeros(self.n, dtype=np.int32)
        for i, t in enumerate(toks):
            u = sorted({tok_id[x] for x in t})
            ids.extend(u)
            ptr[i + 1] = ptr[i] + len(u)
            n_all[i] = len(t)
            b = 0
            for x in u:
                b |= 1 << (((x * 0x9E3779B1) >> 13) & 63)
            sig[i] = b
        self.d_tok_ptr = _to_dev(ptr)
        self.d_tok_ids = _to_dev(np.asarray(ids if ids else [0], dtype=np.int32))
        self.d_sig = _to_dev(sig.view(np.int64), torch.int64)
        self.d_n_all = _to_dev(n_all)

    def ptrs(self):
        out = []
        for b, o in self.dev:
            out += [b, o]
        return out + [self.d_tok_ptr, self.d_tok_ids, self.d_sig, self.d_n_all]


def _enqueue(from_list, to_list, scorer, score_cutoff, exclude_self, n_splits, self_shift, to_index_base, k):
    """Stage both lists (tokens, one vocabulary, the three to-side layouts, one symbol table per alphabet batch) and enqueue
    K3b for every batch and word class: pfz_fuzz_argbest with part_* [n_splits, n_from] when k is None, else pfz_fuzz_topk
    with part_* [n_splits, n_from, k].  Returns (part_idx, part_score, n_splits, staged): `staged` keeps the staged buffers
    alive until the caller has synchronised."""
    dev = _dev()
    n_from, n_to = len(from_list), len(to_list)
    same = to_list is from_list and not to_index_base
    ftoks, fS, fU = _derive(from_list)
    ttoks, tS, tU = (ftoks, fS, fU) if same else _derive(to_list)
    vocab = sorted({x for t in ftoks for x in t} | ({x for t in ttoks for x in t} if not same else set()))
    tok_id = {x: i for i, x in enumerate(vocab)}               # ids in sorted token order: id order == join order of a token set
    tblob, toff, _ = pack_strings(vocab if vocab else [""])
    d_tok_blob = _blob_to_dev(tblob); d_tok_off = _to_dev(toff)
    F = _Side(from_list, ftoks, fS, fU, tok_id)
    T = F if same else _Side(to_list, ttoks, tS, tU, tok_id)
    fl = np.maximum(np.maximum(F.lens[0], F.lens[1]), F.lens[2])
    if len(fl) and fl.max() > MAX_LEN:
        raise ValueError(f"from-string {int(fl.argmax())} has {int(fl.max())} code points; the token / partial scorers "
                         f"support at most {MAX_LEN}")
    # to-side layouts: one length order (by len(b)) for the three variants
    order = np.argsort(T.lens[0], kind="stable").astype(np.int32)
    n_grp = (n_to + 31) // 32
    d_order = _to_dev(order)
    packs = []
    for v in range(3):
        goff = group_word_offsets(T.lens[v][order])
        packs.append((torch.empty(max(int(goff[-1]), 1), dtype=torch.int32, device=dev), _to_dev(goff),
                      torch.empty(n_to, dtype=torch.int32, device=dev)))
    if n_splits is None:
        n_splits = default_splits(n_from, n_grp)
    n_splits = max(1, min(int(n_splits), n_grp))
    shape = (n_splits, n_from) if k is None else (n_splits, n_from, k)
    part_idx = torch.full(shape, -1, dtype=torch.int32, device=dev)
    part_score = torch.zeros(shape, dtype=torch.float64, device=dev)
    counter = torch.zeros(n_splits, dtype=torch.int32, device=dev)
    classes = word_class(fl)
    fblob, foff = F.host[0]
    keep = []
    for lo, hi in _alphabet_batches(fblob, foff):
        cps = np.unique(np.concatenate([fblob[foff[lo]:foff[hi]].astype(np.int64), np.array([0x20], dtype=np.int64)]))
        if len(cps) > 255:
            raise ValueError("a batch of from-strings has more than 254 distinct code points besides the space")
        d_table = _to_dev(symbol_table(cps)); keep.append(d_table)
        for v in range(3):
            _lib.call("pfz_lev_pack", _p(T.dev[v][0]), _p(T.dev[v][1]), _p(d_order), n_to, _p(d_table), _p(packs[v][1]), _p(packs[v][0]),
                      _p(packs[v][2]), _stream())
        for nw in (1, 2, 4, 8, 16):
            ids = np.nonzero(classes[lo:hi] == nw)[0].astype(np.int32) + lo
            if len(ids) == 0:
                continue
            d_ids = _to_dev(ids); keep.append(d_ids)
            tens = F.ptrs() + T.ptrs() + [d_ids, d_table]
            for v in range(3):
                tens += [packs[v][0], packs[v][1], packs[v][2]]
            tens += [d_order, d_tok_blob, d_tok_off, part_idx, part_score, counter, None]
            arr = (ctypes.c_void_p * len(tens))(*[t.data_ptr() if t is not None else 0 for t in tens])
            if k is None:
                _lib.call("pfz_fuzz_argbest", arr, len(tens), n_from, len(ids), int(nw), n_to, SCORER[scorer], float(score_cutoff),
                          int(bool(exclude_self)), int(self_shift), n_splits, _stream())
            else:
                _lib.call("pfz_fuzz_topk", arr, len(tens), n_from, len(ids), int(nw), n_to, SCORER[scorer], float(score_cutoff),
                          int(bool(exclude_self)), int(self_shift), n_splits, int(k), _stream())
    return part_idx, part_score, n_splits, (F, T, packs, keep, d_order, d_tok_blob, d_tok_off)


def fuzz_argbest(from_list, to_list, scorer="WRatio", score_cutoff=0.0, exclude_self=False, n_splits=None, self_shift=0,
                 to_index_base=0):
    """Best to-string per from-string under a rapidfuzz scorer (scores in [0, 100]).  Returns device tensors
    (best_idx int32[n_from] (-1: no to-string reached score_cutoff), best_score float64[n_from]).
    exclude_self skips to-row == from-row + self_shift; to_index_base is added to the returned indices (row-block shards)."""
    if scorer not in SCORER:
        raise NotImplementedError(f"scorer {scorer!r} has no GPU implementation (supported: {sorted(SCORER)})")
    dev = _dev()
    n_from, n_to = len(from_list), len(to_list)
    best_idx = torch.full((max(n_from, 1),), -1, dtype=torch.int32, device=dev)
    best_score = torch.zeros(max(n_from, 1), dtype=torch.float64, device=dev)
    if n_from == 0 or n_to == 0:
        return best_idx[:n_from], best_score[:n_from]
    part_idx, part_score, n_splits, staged = _enqueue(from_list, to_list, scorer, score_cutoff, exclude_self, n_splits, self_shift,
                                                      to_index_base, None)
    part_dist = torch.full((n_splits, n_from), -1, dtype=torch.int32, device=dev)
    best_dist = torch.empty(max(n_from, 1), dtype=torch.int32, device=dev)
    _lib.call("pfz_lev_merge", _p(part_idx), _p(part_score), _p(part_dist), n_splits, n_from, _p(best_idx), _p(best_score), _p(best_dist),
              _stream())
    torch.cuda.current_stream().synchronize()                  # the staged host buffers above go out of scope with this call
    if to_index_base:
        best_idx = torch.where(best_idx >= 0, best_idx + int(to_index_base), best_idx)
    return best_idx[:n_from], best_score[:n_from]


def fuzz_topk(from_list, to_list, k, scorer="WRatio", score_cutoff=0.0, exclude_self=False, n_splits=None, self_shift=0,
              to_index_base=0):
    """The k best to-strings per from-string (1 <= k <= 32) under the candidates and key of fuzz_argbest (score desc, index asc).
    Returns device tensors (idx int32[n_from, k] (-1: empty slot), score float64[n_from, k] (0.0 in empty slots));
    exclude_self, self_shift and to_index_base as in fuzz_argbest."""
    k = check_top_n(k)
    if scorer not in SCORER:
        raise NotImplementedError(f"scorer {scorer!r} has no GPU implementation (supported: {sorted(SCORER)})")
    dev = _dev()
    n_from, n_to = len(from_list), len(to_list)
    if n_from == 0 or n_to == 0:
        return (torch.full((n_from, k), -1, dtype=torch.int32, device=dev), torch.zeros((n_from, k), dtype=torch.float64, device=dev))
    part_idx, part_score, n_splits, staged = _enqueue(from_list, to_list, scorer, score_cutoff, exclude_self, n_splits, self_shift,
                                                      to_index_base, k)
    idx, score = (part_idx[0], part_score[0]) if n_splits == 1 else topk_merge(part_idx, part_score, k)
    torch.cuda.current_stream().synchronize()                  # the staged host buffers above go out of scope with this call
    if to_index_base:
        idx = torch.where(idx >= 0, idx + int(to_index_base), idx)
    return idx, score
