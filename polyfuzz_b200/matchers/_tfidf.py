"""TFIDF matcher -- drop-in for polyfuzz.models.TFIDF (polyfuzz/models/_tfidf.py:11-146) running the
vectoriser (K1) and the sparse cosine top-n (K2) on an H100, on one GPU or many through the same driver
(distributed.tfidf_topk_sharded)."""
from typing import List, Tuple

import numpy as np
import pandas as pd

from ._base import BaseMatcher
from ._utils import (arrow_from_staged, assemble_matches, assemble_matches_device, clip_top_n, device_tail_available,
                     prepare_strings)
from .. import engine
from ..distributed import gather_string_shards, get_comm, shard_bounds, tfidf_topk_sharded
from ..strings import ARROW_CACHE


class TFIDF(BaseMatcher):
    """
    A character based n-gram TF-IDF to approximate edit distance (same constructor as the reference).

    Arguments:
        n_gram_range: The n_gram_range on a character-level
        clean_string: Whether to clean the string such that only alphanumerical characters are kept
        min_similarity: The minimum similarity between strings, otherwise return 0 similarity
        top_n: The number of matches you want returned
        cosine_method: "sparse" | "sklearn" | "knn".  Every value runs the same fused GPU kernel; what
                       differs is the reference branch whose semantics are reproduced: `sparse` keeps
                       only candidates with score > min_similarity (polyfuzz/models/_utils.py:82), while
                       the reference's `sklearn` and `knn` branches never look at min_similarity
                       (_utils.py:59-70, 94-102: every to-string is ranked, scores below 0.001 are blanked
                       afterwards) -- here: the kernel threshold is 0 for those two methods.
        model_id: The name of the particular instance, used when comparing models
        remove_space_ngrams: Remove n-grams that contain a space
        distributed: (new) when True and torch.distributed is initialised with world size > 1
                     (torchrun, one process per GPU), every rank calls match() with the SAME lists;
                     the to_list is sharded in contiguous row-blocks, per-shard top-k lists are
                     exchanged with one NCCL all-gather and merged; all ranks return the same frame.
    """

    def __init__(self,
                 n_gram_range: Tuple[int, int] = (3, 3),
                 clean_string: bool = True,
                 min_similarity: float = 0.75,
                 top_n: int = 1,
                 cosine_method: str = "sparse",
                 model_id: str = None,
                 remove_space_ngrams=True,
                 distributed: bool = False):
        super().__init__(model_id)
        self.type = "TF-IDF"
        self.n_gram_range = n_gram_range
        self.clean_string = clean_string
        self.min_similarity = min_similarity
        self.cosine_method = cosine_method
        self.top_n = top_n
        self.vectorizer = None
        self.tf_idf_to = None
        self.remove_space_ngrams = remove_space_ngrams
        self.distributed = distributed
        self._index = None              # device inverted index of tf_idf_to (rebuilt lazily after unpickling)
        self._shard = (0, 0)            # [lo, hi) to-rows owned by this rank (all of them on one GPU)
        self._st_to = None              # device-resident to-list (blob, offsets) for the frame tail; not pickled
        self._st_from = None            # ... and the from-rows of the current call

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_index"] = None
        st["_st_to"] = st["_st_from"] = None
        if self.tf_idf_to is not None and not hasattr(self.tf_idf_to, "tocsr"):
            st["tf_idf_to"] = self.tf_idf_to.to_scipy()          # device CSR -> host scipy for joblib.dump
        return st

    def match(self, from_list: List[str], to_list: List[str] = None, re_train: bool = True,
              from_block: Tuple[int, int] = None) -> pd.DataFrame:
        """Match two lists of strings to each other and return the most similar strings
        (polyfuzz/models/_tfidf.py:68-100).

        from_block=(lo, hi) (new, self-match only): return the matches of from_list[lo:hi] against the
        whole from_list (diagonal excluded) -- one row-block of a self-match that is too large for one
        call / one GPU; the frame has hi-lo rows."""
        ARROW_CACHE.clear()
        self._st_from = None
        top_idx, top_val, top_n = self.match_arrays(from_list, to_list, re_train, from_block)     # kernels are in flight
        st_from, st_to = self._st_from, self._st_to
        self._st_from = None
        if top_idx.shape[0] > 0 and st_to is not None and device_tail_available(st_from) and st_to[2]:
            # K5: rounding, blanking and the per-rank string gathers on the device; the host wraps the finished columns
            return assemble_matches_device(arrow_from_staged(st_from), st_to[0], st_to[1], top_idx, top_val)
        rows = from_list if from_block is None else from_list[from_block[0]:from_block[1]]
        targets = to_list if to_list is not None else from_list
        prepared = prepare_strings(rows, targets if (to_list is not None or from_block is not None) else None)   # overlaps the GPU
        out = assemble_matches(rows, targets, top_idx.cpu().numpy(), top_val.cpu().numpy(), prepared=prepared)
        ARROW_CACHE.clear()
        return out

    def _threshold(self):
        """Kernel threshold of the reproduced reference branch (see cosine_method in the class docstring)."""
        if self.cosine_method in ("sklearn", "knn"):
            return 0.0
        if self.cosine_method != "sparse":
            raise ValueError(f"cosine_method {self.cosine_method!r} unknown (sparse | sklearn | knn)")
        return self.min_similarity

    def match_arrays(self, from_list, to_list=None, re_train=True, from_block=None):
        """Device-side result: (top_idx int32[n,k] with -1 for no match, top_val float64[n,k], k).
        One GPU or many, the lists are staged here and scored by one driver (distributed.tfidf_topk_sharded)."""
        top_n = clip_top_n(self.top_n, to_list)
        if top_n < 1:
            raise ValueError("top_n must be >= 1 and to_list must not be empty")
        from_base, rows = 0, from_list
        if from_block is not None:
            if to_list is not None:
                raise ValueError("from_block is only meaningful for a self-match (to_list=None)")
            lo, hi = int(from_block[0]), int(from_block[1])
            if not (0 <= lo <= hi <= len(from_list)):
                raise ValueError(f"from_block {from_block} out of range")
            from_base, rows = lo, from_list[lo:hi]
        threshold = self._threshold()
        if re_train:
            self.vectorizer = engine.NgramTfidf(self.n_gram_range, self.clean_string, self.remove_space_ngrams)
        elif self.vectorizer is None or self.tf_idf_to is None:
            raise ValueError("re_train=False needs a fitted model (call match/fit first)")
        vec = self.vectorizer
        comm = get_comm() if self.distributed else None
        full_to = to_list if to_list else from_list          # `if to_list:` as in _tfidf.py:107
        staged_to = None
        if re_train:
            self._shard = shard_bounds(len(full_to), comm.world_size, comm.rank) if comm else (0, len(full_to))
            lo, hi = self._shard
            staged_to = vec.stage(full_to[lo:hi] if comm else full_to)
            # the frame tail needs every to-string on every rank: the shards' blobs are all-gathered over NCCL (bytes), so the
            # host work per rank stays that of its own shard
            self._st_to = gather_string_shards(comm, staged_to) if comm else self._tail_of(staged_to)
        if comm is None and not to_list and from_block is None:
            # one GPU, whole self-match: the to-list is the from-list (polyfuzz/models/_tfidf.py:114-116); a transform
            # scores the fitted to-matrix itself instead of vectorising the list again
            staged_from = staged_to if re_train else self._device_to()
            self._st_from = staged_to if re_train else (self._st_to[3] if self._st_to is not None else None)
        else:
            staged_from = self._st_from = vec.stage(rows)
        if not re_train and self._index is None:             # restored from a pickle: the index is rebuilt from the to-matrix
            self._index = engine.index_for(self._device_to(), vec)
        idx, val, csr_to, self._index = tfidf_topk_sharded(vec, staged_from, staged_to, self._shard[0], top_n, threshold,
                                                           to_list is None, from_base, fit=re_train, fit_on_from=bool(to_list),
                                                           comm=comm, index=self._index,
                                                           n_docs_total=len(full_to) + (len(from_list) if to_list else 0))
        if re_train:
            self.tf_idf_to = csr_to
        return idx, val, top_n

    @staticmethod
    def _tail_of(S):
        """(device blob int32, device offsets int64, ascii?, staged list) of a to-list kept for the frame tail (K5)."""
        return (S.d_blob, S.d_off, bool(S.ascii), S)

    def _device_to(self):
        if hasattr(self.tf_idf_to, "tocsr"):                      # restored from a pickle
            self.tf_idf_to = engine.CsrMatrix.from_scipy(self.tf_idf_to)
        return self.tf_idf_to
