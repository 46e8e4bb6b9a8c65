"""RapidFuzz / EditDistance matchers -- drop-ins for polyfuzz.models.RapidFuzz
(polyfuzz/models/_rapidfuzz.py:11-113) and polyfuzz.models.EditDistance
(polyfuzz/models/_distance.py:12-102) whose all-pairs scoring runs on the GPU (K3 / K3b).

Scorers (rapidfuzz 3.x definitions, no preprocessing -- oracle/fuzz.py restates them and is pinned on rapidfuzz's
published known answers):
  * "WRatio" (the reference's default for RapidFuzz, fuzz.WRatio, _rapidfuzz.py:48), "QRatio", "partial_ratio",
    "token_sort_ratio", "token_set_ratio", "token_ratio", "partial_token_sort_ratio", "partial_token_set_ratio",
    "partial_token_ratio"                                         -> csrc/pfz_fuzz.cu (K3b)
  * "ratio" (fuzz.ratio, the reference's default for EditDistance, _distance.py:32) and "levenshtein"
    (Levenshtein.normalized_similarity)                                  -> csrc/pfz_lev.cu (K3)
  * EditDistance only: "jaro_similarity" / "jaro" and "jaro_winkler_similarity" / "jaro_winkler" (jellyfish's
    definitions with long_tolerance=False, the custom scorer of the reference's tutorial; raw 0..1 scores)
                                                                         -> csrc/pfz_lev.cu (K3, Jaro mode)
  * "osa" / "optimal_string_alignment" / "osa_normalized_similarity" (rapidfuzz.distance.OSA.normalized_similarity: optimal
    string alignment, i.e. restricted Damerau-Levenshtein -- a swap of two adjacent characters is one edit, no substring is
    edited twice, so "CA" -> "ABC" costs 3, not unrestricted Damerau-Levenshtein's 2; 0..1 scores like "levenshtein")
                                                                         -> csrc/pfz_lev.cu (K3, OSA mode)
  * "dl" / "unrestricted_damerau_levenshtein" / "damerau_levenshtein_normalized_similarity" (unrestricted Damerau-Levenshtein,
    rapidfuzz.distance.DamerauLevenshtein's metric: a swapped pair may be edited again, so "CA" -> "ABC" costs 2;
    1 - dl / max(|a|, |b|), 0..1 scores like "levenshtein")             -> csrc/pfz_lev.cu (K3, dl_kernel, gated by OSA)
  * rapidfuzz.distance's other normalised similarities, 1 - d / M on 0..1 like "levenshtein" (DESIGN.md 4.18):
    "indel" / "indel_normalized_similarity" (d = |a| + |b| - 2 LCS, M = |a| + |b|: fuzz.ratio / 100 without the rounding of the
    round trip), "lcsseq" / "lcs_seq" / "lcsseq_normalized_similarity" / "lcs_seq_normalized_similarity" (d = M - LCS),
    "hamming" / "hamming_normalized_similarity" (rapidfuzz 3's pad=True: unequal lengths count the surplus as mismatches, where
    rapidfuzz 2 raises), "prefix" / "prefix_normalized_similarity" and "postfix" / "postfix_normalized_similarity" (d = M - the
    common prefix / suffix length); M = max(|a|, |b|) but for Indel
                                                                         -> csrc/pfz_lev.cu (K3, lev_kernel's LCS / pos_kernel)
  * functools.partial(<a callable that resolves to "levenshtein">, weights=(insertion, deletion, substitution)) -- rapidfuzz's
    Levenshtein.normalized_similarity(from, to, weights=...): weighted Levenshtein, 1 - D / M on 0..1 like "levenshtein",
    each weight an int in [0, 65535] (anything else is a ValueError); (w, w, w) scores as "levenshtein" -> csrc/pfz_lev.cu (K3,
    wlev_kernel; DESIGN.md 4.17).  The partial may carry no positional arguments and no keyword but `weights`; every other
    partial raises NotImplementedError.  A partial of DamerauLevenshtein.normalized_similarity resolves as Levenshtein (the rule
    below), so it scores weighted Levenshtein where rapidfuzz itself would reject `weights`.
The bare name "damerau_levenshtein" raises NotImplementedError: some libraries mean OSA by it, others unrestricted DL, so the
user picks "osa" or "dl".
A scorer may be given by name or as the rapidfuzz / jellyfish callable of that __name__.  A callable named
`normalized_similarity` is OSA when a dotted component of its __module__ is "osa" or starts with "osa_" (case-insensitive, e.g.
rapidfuzz.distance.OSA), and normalised Levenshtein otherwise -- including rapidfuzz.distance.DamerauLevenshtein's, Indel's,
LCSseq's, Hamming's, Prefix's and Postfix's, which therefore score Levenshtein; pointing them at their own metrics changes what an
existing call returns, so it is left to a separate fix, and the names above are the way to these scorers.  These rules are
written from rapidfuzz's documented module layout;
rapidfuzz is not a dependency, so its callables' actual __name__ / __module__ values are not checked by the tests, which use
stand-in functions.  Arbitrary Python callables cannot be compiled to the device and raise NotImplementedError -- there is no
CPU fallback.
top_n = k (1..32) returns the k best to-strings per from-string (process.extract(..., limit=k) semantics: score desc, then
to-index asc) in the columns To, Similarity, To_2, Similarity_2, ...; the reference implements top_n only for TF-IDF and
Embeddings (polyfuzz/polyfuzz.py:100-102).  top_n = 1 is the arg-best path, unchanged.
candidates = TFIDF(...) (new): score only each from-string's TF-IDF candidates -- `candidates.match_arrays(from_list, to_list,
re_train)`, its top-n to-indices per row -- with this matcher's scorer, instead of every pair (blocking, DESIGN.md 4.16).  Each
row is the all-pairs row of the same matcher against the to-strings of its candidate list (same scores, cutoff, key and
self-exclusion), and a row without a candidate that passes is (None, 0.0), for EditDistance too; EditDistance's `normalize`
then takes its min and max over the filled cells, as its top_n > 1 path does.  A to-string outside a row's TF-IDF top-n is
never scored, so the best edit-distance match can be missed: that is the trade (DESIGN.md 7.16 measures it).
Deviations from the reference, both documented reference bugs (SURVEY.md 8a): a self-match excludes
index i only (the reference mutates the shared to_list, _rapidfuzz.py:103-104), and the matcher can be
reused for a two-list call after a self-match (`equal_lists` is per call)."""
import functools
from typing import Callable, List, Union

import numpy as np
import pandas as pd

from ._base import BaseMatcher
from ._utils import clip_top_n
from .. import editdist, fuzzy
from ..distributed import get_comm, merge_topk_any, shard_bounds

_NAMES = {"ratio": "ratio", "levenshtein": "norm_lev", "norm_lev": "norm_lev", "normalized_similarity": "norm_lev",
          "normalized_levenshtein": "norm_lev", "osa": "norm_osa", "optimal_string_alignment": "norm_osa",
          "osa_normalized_similarity": "norm_osa", "dl": "norm_dl", "unrestricted_damerau_levenshtein": "norm_dl",
          "damerau_levenshtein_normalized_similarity": "norm_dl", "indel": "norm_indel", "indel_normalized_similarity": "norm_indel",
          "lcsseq": "norm_lcsseq", "lcs_seq": "norm_lcsseq", "lcsseq_normalized_similarity": "norm_lcsseq",
          "lcs_seq_normalized_similarity": "norm_lcsseq", "hamming": "norm_hamming", "hamming_normalized_similarity": "norm_hamming",
          "prefix": "norm_prefix", "prefix_normalized_similarity": "norm_prefix", "postfix": "norm_postfix",
          "postfix_normalized_similarity": "norm_postfix"}
_FUZZ = {k.lower(): k for k in fuzzy.SCORER if k != "ratio"}
# jellyfish's function names (and short forms); 0..1 scores, so only EditDistance takes them
_JARO = {"jaro": "jaro", "jaro_similarity": "jaro", "jaro_winkler": "jaro_winkler", "jaro_winkler_similarity": "jaro_winkler"}


def _is_osa_module(module) -> bool:
    """rapidfuzz.distance.OSA and its implementation modules (OSA_py, OSA_cpp, ...): a dotted component "osa" or "osa_*"."""
    parts = module.lower().split(".") if isinstance(module, str) else []
    return any(p == "osa" or p.startswith("osa_") for p in parts)


def _resolve_scorer(scorer, default, allow_jaro=False) -> str:
    """-> "ratio" | "norm_lev" | "norm_osa" | "norm_dl" | "jaro" | "jaro_winkler" | "wlev" | one of editdist.SEQ_METRICS (K3) or
    one of fuzzy.SCORER (K3b).
    A functools.partial is "wlev" (weighted Levenshtein, its weights from _scorer_weights) or, with weights None or (w, w, w),
    "norm_lev"."""
    if scorer is None:
        scorer = default
    if isinstance(scorer, functools.partial):
        return "wlev" if editdist.uniform_weight(_scorer_weights(scorer, allow_jaro)) == 0 else "norm_lev"
    key = scorer.lower() if isinstance(scorer, str) else getattr(scorer, "__name__", "").lower()
    if key == "normalized_similarity" and not isinstance(scorer, str) and _is_osa_module(getattr(scorer, "__module__", None)):
        return "norm_osa"
    if key in _NAMES:
        return _NAMES[key]
    if key in _FUZZ:
        return _FUZZ[key]
    if allow_jaro and key in _JARO:
        return _JARO[key]
    if key == "damerau_levenshtein":
        raise NotImplementedError(f"scorer {scorer!r} is ambiguous: use 'osa' (optimal string alignment, restricted "
                                  "Damerau-Levenshtein) or 'dl' (unrestricted Damerau-Levenshtein)")
    raise NotImplementedError(f"scorer {scorer!r} has no GPU implementation (supported: 'ratio', 'levenshtein', 'osa', 'dl', "
                              "'indel', 'lcsseq', 'hamming', 'prefix', 'postfix', "
                              f"{sorted(_FUZZ.values())}" + (", 'jaro_similarity', 'jaro_winkler_similarity'" if allow_jaro else "")
                              + "); polyfuzz_b200 has no CPU fallback")


def _scorer_weights(scorer, allow_jaro=False):
    """The validated `weights` (editdist.check_weights) of a partial scorer, None for any other scorer.  A partial is accepted
    only when its func resolves to "norm_lev" by _resolve_scorer's rules and it has no positional arguments and no keyword
    but `weights`; otherwise NotImplementedError."""
    if not isinstance(scorer, functools.partial):
        return None
    try:
        base = _resolve_scorer(scorer.func, None, allow_jaro)
    except NotImplementedError:
        base = None
    if base != "norm_lev" or scorer.args or not set(scorer.keywords) <= {"weights"}:
        raise NotImplementedError(f"scorer {scorer!r} has no GPU implementation: a functools.partial is supported only as a "
                                  "partial of Levenshtein.normalized_similarity with the keyword `weights` and no other "
                                  "argument; polyfuzz_b200 has no CPU fallback")
    return editdist.check_weights(scorer.keywords.get("weights"))


def _argbest(from_list, targets, metric, cutoff, self_match, distributed, kept=None, reuse=False, weights=None):
    """Best to-string per from-string on this GPU, or -- distributed=True under torchrun -- on the to_list row-block of every
    rank followed by ONE all-gather of the per-shard bests and the canonical merge (score desc, global index asc): all ranks
    get the single-GPU result (SURVEY.md 8e; the reference's own fan-out is per from-row, polyfuzz/models/_rapidfuzz.py:92-95).
    kept / reuse: the matcher's kept to-side (editdist.KeptTargets; each rank keeps its own shard) and whether it may serve
    this call.  metric "wlev" scores weighted Levenshtein with `weights`."""
    comm = get_comm() if distributed else None
    token_scorer = metric in fuzzy.SCORER and metric != "ratio"
    if comm is None:
        if token_scorer:
            return fuzzy.fuzz_argbest(from_list, targets, metric, cutoff, exclude_self=self_match, kept=kept, reuse=reuse) + (None,)
        if metric == "wlev":
            return editdist.edit_wlev_argbest(from_list, targets, weights, cutoff, exclude_self=self_match, kept=kept, reuse=reuse)
        return editdist.edit_argbest(from_list, targets, metric, cutoff, exclude_self=self_match, kept=kept, reuse=reuse)
    lo, hi = shard_bounds(len(targets), comm.world_size, comm.rank)
    if token_scorer:
        bi, bs = fuzzy.fuzz_argbest(from_list, targets[lo:hi], metric, cutoff, exclude_self=self_match, self_shift=-lo, to_index_base=lo,
                                    kept=kept, reuse=reuse)
        bd = torch_full_like_int(bi)
    else:
        Q = editdist.EditQueries(from_list)
        T = _shard_targets(targets[lo:hi], lo, kept, reuse)
        if metric == "wlev":
            bi, bs, bd = editdist.edit_wlev_argbest_staged(Q, T, weights, cutoff, exclude_self=self_match, self_shift=-lo,
                                                           to_index_base=lo)
        else:
            bi, bs, bd = editdist.edit_argbest_staged(Q, T, metric, cutoff, exclude_self=self_match, self_shift=-lo, to_index_base=lo)
    gi, gs, gd = comm.all_gather_best(bi, bs, bd)
    return editdist.lev_merge(gi, gs, gd)


def _shard_targets(shard, lo, kept, reuse):
    """This rank's staged K3 to-shard: the kept one when it may serve, else a new EditTargets (kept when a holder is given)."""
    if kept is None:
        return editdist.EditTargets(shard)
    return kept.stage(("k3", lo), shard, lambda lst: editdist.EditTargets(lst), reuse)


def _topk(from_list, targets, metric, cutoff, self_match, distributed, k, kept=None, reuse=False, weights=None):
    """Top-k sibling of _argbest: the k best to-strings per from-string (device idx int32[n, k], -1 = empty slot, and score
    float64[n, k]) on this GPU, or -- distributed=True under torchrun -- per to_list row-block followed by ONE all-gather of the
    per-shard lists and the canonical merge, as TF-IDF and Embeddings do: all ranks get the single-GPU result."""
    comm = get_comm() if distributed else None
    token_scorer = metric in fuzzy.SCORER and metric != "ratio"
    if comm is None:
        if token_scorer:
            return fuzzy.fuzz_topk(from_list, targets, k, metric, cutoff, exclude_self=self_match, kept=kept, reuse=reuse)
        if metric == "wlev":
            return editdist.edit_wlev_topk(from_list, targets, k, weights, cutoff, exclude_self=self_match, kept=kept, reuse=reuse)
        return editdist.edit_topk(from_list, targets, k, metric, cutoff, exclude_self=self_match, kept=kept, reuse=reuse)
    lo, hi = shard_bounds(len(targets), comm.world_size, comm.rank)
    if token_scorer:
        idx, val = fuzzy.fuzz_topk(from_list, targets[lo:hi], k, metric, cutoff, exclude_self=self_match, self_shift=-lo, to_index_base=lo,
                                   kept=kept, reuse=reuse)
    else:
        Q = editdist.EditQueries(from_list)
        T = _shard_targets(targets[lo:hi], lo, kept, reuse)
        if metric == "wlev":
            idx, val = editdist.edit_wlev_topk_staged(Q, T, k, weights, cutoff, exclude_self=self_match, self_shift=-lo,
                                                      to_index_base=lo)
        else:
            idx, val = editdist.edit_topk_staged(Q, T, k, metric, cutoff, exclude_self=self_match, self_shift=-lo, to_index_base=lo)
    gi, gv = comm.all_gather_topk(idx.contiguous(), val.contiguous())
    return merge_topk_any(gi, gv, k)


def _topk_frame(from_list, targets, idx, score):
    """From, To, Similarity, To_2, Similarity_2, ... from host top-k arrays; scores unrounded, an empty slot is (None, 0.0)."""
    to_arr = np.empty(len(targets) + 1, dtype=object); to_arr[:-1] = targets; to_arr[-1] = None
    cols = {"From": pd.Series(list(from_list), dtype=object)}
    for r in range(idx.shape[1]):
        filled = idx[:, r] >= 0
        cols["To" if r == 0 else f"To_{r + 1}"] = pd.Series(to_arr[np.where(filled, idx[:, r], len(targets))], dtype=object)
        cols["Similarity" if r == 0 else f"Similarity_{r + 1}"] = np.where(filled, score[:, r], 0.0)
    return pd.DataFrame(cols)


def _check_candidates(candidates, top_n, distributed):
    """The constructors' check of `candidates`: None, or a TFIDF with top_n >= the matcher's and distributed=False (the TF-IDF
    itself may be distributed: its merged top-n is the same on every rank)."""
    if candidates is None:
        return None
    from ._tfidf import TFIDF
    if not isinstance(candidates, TFIDF):
        raise ValueError(f"candidates must be a polyfuzz_b200.TFIDF instance, got {type(candidates).__name__}")
    if top_n > candidates.top_n:
        raise ValueError(f"top_n={top_n} exceeds the candidates' top_n={candidates.top_n}")
    if distributed:
        raise ValueError("distributed=True cannot be combined with candidates: each rank scores the few candidate pairs itself "
                         "(pass distributed=True to the TFIDF instead)")
    return candidates


def _cand_topk(from_list, targets, metric, cutoff, self_match, k, candidates, to_list, re_train, kept, weights=None):
    """Candidate mode: TF-IDF's device top-n of every from-string, then the k best of those under the matcher's scorer.
    Returns host (idx int32[n, k], -1 = empty slot, score float64[n, k])."""
    cand, _, _ = candidates.match_arrays(from_list, to_list, re_train)
    token_scorer = metric in fuzzy.SCORER and metric != "ratio"
    if token_scorer:
        idx, score = fuzzy.fuzz_cand_topk(from_list, targets, cand, k, metric, cutoff, exclude_self=self_match, kept=kept,
                                          reuse=not re_train)
    elif metric == "wlev":
        idx, score = editdist.edit_wlev_cand_topk(from_list, targets, cand, k, weights, cutoff, exclude_self=self_match, kept=kept,
                                                  reuse=not re_train)[:2]
    else:
        idx, score = editdist.edit_cand_topk(from_list, targets, cand, k, metric, cutoff, exclude_self=self_match, kept=kept,
                                             reuse=not re_train)[:2]
    idx = idx.cpu().numpy(); score = score.cpu().numpy()
    return (idx[:, None], score[:, None]) if k == 1 else (idx, score)


def torch_full_like_int(t):
    import torch
    return torch.full_like(t, -1)


class _KeepsTargets:
    """A matcher that keeps the to-side it staged last (editdist.KeptTargets): a call with re_train=False whose to-list equals
    the kept one (same length, == element by element) scores against it without staging it again -- PolyFuzz.transform's
    `match(new, self.to_list, re_train=False)`.  A self-match's list counts as its to-list.  Pickling drops the device state;
    the first call after loading stages again."""

    def _kept(self):
        kept = self.__dict__.get("_kept_targets")
        if kept is None:
            kept = self._kept_targets = editdist.KeptTargets()
        return kept

    def _weights_kw(self):
        """The weighted-Levenshtein weights for _argbest / _topk / _cand_topk, passed only when the metric is "wlev"."""
        return {"weights": self._weights} if self._metric == "wlev" else {}

    def __getstate__(self):
        st = dict(self.__dict__)
        st.pop("_kept_targets", None)
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)

class RapidFuzz(_KeepsTargets, BaseMatcher):
    """Edit-distance matcher (GPU).  Arguments as in the reference: n_jobs (accepted, ignored -- the GPU
    scores all pairs in one launch), score_cutoff in [0,1], scorer (default fuzz.WRatio, as the reference), model_id.
    top_n (1..32): matches per from-string, clipped to the number of distinct to-strings when a to_list is given.
    candidates (a TFIDF, top_n >= this top_n): score only its candidates per from-string (see the module docstring)."""

    def __init__(self, n_jobs: int = 1, score_cutoff: float = 0, scorer: Union[str, Callable] = "WRatio", model_id: str = None,
                 distributed: bool = False, top_n: int = 1, candidates=None):
        super().__init__(model_id)
        self.top_n = editdist.check_top_n(top_n)
        self.candidates = _check_candidates(candidates, self.top_n, distributed)
        self.type = "EditDistance"
        self.distributed = distributed
        self.score_cutoff = score_cutoff * 100
        self.scorer = scorer
        self._metric = _resolve_scorer(scorer, "WRatio")
        self._weights = _scorer_weights(scorer)
        self.equal_lists = False
        self.n_jobs = n_jobs

    def match(self, from_list: List[str], to_list: List[str] = None, re_train: bool = True, **kwargs) -> pd.DataFrame:
        """(from, best to, score/100); no candidate with score >= score_cutoff -> (from, None, 0.0)
        (polyfuzz/models/_rapidfuzz.py:106-113).  top_n > 1: the k best, an empty slot is (None, 0.0).
        re_train=False: score against the kept to-side when to_list equals the list it was staged from (the frame is the
        same as a fresh call's); any call that stages keeps its to-side."""
        self_match = to_list is None
        targets = from_list if self_match else to_list
        unit = self._metric in ("norm_lev", "norm_osa", "norm_dl", "wlev") + editdist.SEQ_METRICS     # scores already on 0..1
        scale = 1.0 if unit else 100.0
        cutoff = self.score_cutoff / 100.0 if unit else self.score_cutoff
        top_n = clip_top_n(self.top_n, to_list)
        if getattr(self, "candidates", None) is not None:
            idx, score = _cand_topk(from_list, targets, self._metric, cutoff, self_match, top_n, self.candidates, to_list, re_train,
                                    self._kept(), **self._weights_kw())
            return _topk_frame(from_list, targets, idx, score / scale)
        if top_n > 1:
            idx, score = _topk(from_list, targets, self._metric, cutoff, self_match, self.distributed, top_n, self._kept(), not re_train,
                               **self._weights_kw())
            return _topk_frame(from_list, targets, idx.cpu().numpy(), score.cpu().numpy() / scale)
        idx, score, _ = _argbest(from_list, targets, self._metric, cutoff, self_match, self.distributed, self._kept(), not re_train,
                                 **self._weights_kw())
        idx = idx.cpu().numpy(); score = score.cpu().numpy() / scale
        to_arr = np.empty(len(targets) + 1, dtype=object); to_arr[:-1] = targets; to_arr[-1] = None
        sel = np.where(idx >= 0, idx, len(targets))
        return pd.DataFrame({"From": pd.Series(list(from_list), dtype=object), "To": pd.Series(to_arr[sel], dtype=object),
                             "Similarity": np.where(idx >= 0, score, 0.0)})


def _normalize_filled(idx, score):
    """EditDistance's min-max normalisation over the filled cells (idx >= 0) of a top-k frame; empty slots stay 0.0."""
    filled = idx >= 0
    if not filled.any():
        return np.zeros_like(score)
    lo, hi = score[filled].min(), score[filled].max()
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(filled, (score - lo) / (hi - lo), 0.0)


class EditDistance(_KeepsTargets, BaseMatcher):
    """Edit-distance matcher with the reference's EditDistance surface (n_jobs, scorer, model_id, normalize):
    Similarity is the scorer's raw value (fuzz.ratio: 0..100, Levenshtein / weighted Levenshtein / OSA / DL / Jaro / Jaro-Winkler:
    0..1) of the best to-string,
    min-max normalised over the column when `normalize` (polyfuzz/models/_distance.py:83-86).
    top_n (1..32): matches per from-string, clipped to the number of distinct to-strings when a to_list is given; an empty
    slot is (None, 0.0).  With top_n > 1, `normalize` takes ONE min and ONE max over every filled Similarity cell of the
    frame (empty slots excluded), so the first Similarity column can differ from the top_n = 1 frame's, whose min and max
    cover the best matches only; without `normalize` the first three columns are the top_n = 1 frame.
    candidates (a TFIDF, top_n >= this top_n): score only its candidates per from-string (see the module docstring).
    scorer may be functools.partial(Levenshtein.normalized_similarity, weights=(insertion, deletion, substitution)), rapidfuzz's
    weighted Levenshtein (the one way to pass a rapidfuzz keyword through the reference's scorer(a, b) interface); see the module
    docstring for the rules."""

    def __init__(self, n_jobs: int = 1, scorer: Union[str, Callable] = "ratio", model_id: str = None, normalize: bool = True,
                 distributed: bool = False, top_n: int = 1, candidates=None):
        super().__init__(model_id)
        self.top_n = editdist.check_top_n(top_n)
        self.candidates = _check_candidates(candidates, self.top_n, distributed)
        self.type = "EditDistance"
        self.distributed = distributed
        self.scorer = scorer
        self._metric = _resolve_scorer(scorer, "ratio", allow_jaro=True)
        self._weights = _scorer_weights(scorer, allow_jaro=True)
        self.normalize = normalize
        self.equal_lists = False
        self.n_jobs = n_jobs

    def match(self, from_list: List[str], to_list: List[str] = None, re_train: bool = True, **kwargs) -> pd.DataFrame:
        """re_train as in RapidFuzz.match."""
        self_match = to_list is None
        targets = from_list if self_match else to_list
        if len(targets) - (1 if self_match else 0) < 1:
            raise ValueError("attempt to get argmax of an empty sequence")         # np.argmax on [] in the reference
        # np.argmax over the scorer's values (polyfuzz/models/_distance.py:98-99): no cutoff; the token scorers take
        # score_cutoff = 0 (their default), which every score passes
        no_cut = 0.0 if self._metric in fuzzy.SCORER and self._metric != "ratio" else float("-inf")
        top_n = clip_top_n(self.top_n, to_list)
        cand = getattr(self, "candidates", None) is not None
        if top_n > 1 or cand:
            if cand:
                idx, score = _cand_topk(from_list, targets, self._metric, no_cut, self_match, top_n, self.candidates, to_list,
                                        re_train, self._kept(), **self._weights_kw())
            else:
                idx, score = _topk(from_list, targets, self._metric, no_cut, self_match, self.distributed, top_n, self._kept(),
                                   not re_train, **self._weights_kw())
                idx = idx.cpu().numpy(); score = score.cpu().numpy()
            return _topk_frame(from_list, targets, idx, _normalize_filled(idx, score) if self.normalize else score)
        idx, score, _ = _argbest(from_list, targets, self._metric, no_cut, self_match, self.distributed, self._kept(), not re_train,
                                 **self._weights_kw())
        idx = idx.cpu().numpy(); score = score.cpu().numpy()
        to_arr = np.empty(len(targets), dtype=object); to_arr[:] = targets
        matches = pd.DataFrame({"From": pd.Series(list(from_list), dtype=object), "To": pd.Series(to_arr[idx], dtype=object),
                                "Similarity": score})
        if self.normalize:
            s = matches["Similarity"]
            matches["Similarity"] = (s - s.min()) / (s.max() - s.min())
        return matches
