"""Embeddings matcher -- drop-in for the pre-computed-vector path of polyfuzz.models.Embeddings
(polyfuzz/models/_embeddings.py:87-135): dense cosine top-n on the tensor cores (K4).  The language-model
embedders themselves (`_embed`, Flair / SBERT / ...) are out of scope (SURVEY.md section 2, rows 7-8): supply
`embeddings_from` / `embeddings_to`, or an `embedding_method` callable `list[str] -> ndarray`.

precision="bf16" (default) ranks bf16-rounded rows on fp32 tensor-core accumulators; precision="fp64" returns the canonical
fp64 cosine top-n bit for bit (DESIGN.md 2 and 4.6), the reference's sklearn-branch scores up to the last bits.  Any top_n
works in both precisions: above 32 the rows take a bound pass, a threshold pass and a select on the GPU (DESIGN.md 4.7), with
the same results as the top-k kernel would give; the only limit is memory for the n_from x top_n result."""
from typing import Callable, List

import numpy as np
import pandas as pd

from ._base import BaseMatcher
from ._utils import assemble_matches, clip_top_n
from .. import dense
from ..distributed import get_comm, merge_topk_any, shard_bounds


class Embeddings(BaseMatcher):
    def __init__(self, embedding_method: Callable = None, min_similarity: float = 0.75, top_n: int = 1,
                 cosine_method: str = "sparse", model_id: str = None, distributed: bool = False, precision: str = "bf16"):
        super().__init__(model_id)
        if precision not in ("bf16", "fp64"):
            raise ValueError(f"precision {precision!r} unknown (bf16 | fp64)")
        self.precision = precision
        self.type = "Embeddings"
        self.distributed = distributed      # torchrun: the to-matrix is row-sharded, one all-gather of per-shard top-k + merge
        self.embedding_method = embedding_method
        self.min_similarity = min_similarity
        self.top_n = top_n
        self.cosine_method = cosine_method
        self.embeddings_to = None

    def _embed(self, strings):
        if not callable(self.embedding_method):
            raise NotImplementedError("language-model embedders are out of scope here: pass embeddings_from / embeddings_to "
                                      "or an embedding_method callable (list[str] -> ndarray)")
        return np.asarray(self.embedding_method(strings))

    def match(self, from_list: List[str], to_list: List[str] = None, embeddings_from: np.ndarray = None,
              embeddings_to: np.ndarray = None, re_train: bool = True) -> pd.DataFrame:
        """polyfuzz/models/_embeddings.py:87-135.  Rows are l2-normalised (as the reference's sklearn branch does,
        sk:metrics/pairwise.py:1744-1750; identical to its sparse branch for unit-norm inputs)."""
        given = lambda e: isinstance(e, np.ndarray)            # noqa: E731
        vec_from = embeddings_from if given(embeddings_from) else self._embed(from_list)
        if given(embeddings_to):
            vec_to = embeddings_to
        elif not re_train:
            vec_to = self.embeddings_to                          # fitted earlier (PolyFuzz.transform)
            if vec_to is None:
                raise ValueError("re_train=False needs embeddings from an earlier match/fit")
        else:
            vec_to = vec_from if to_list is None else self._embed(to_list)
        embeddings_from, embeddings_to = vec_from, vec_to
        top_n = clip_top_n(self.top_n, to_list)
        comm = get_comm() if self.distributed else None
        exact = self.precision == "fp64"
        stage = dense.stage_exact if exact else (lambda e: dense.to_bf16_rows(e, normalize=True)[0])
        x = stage(embeddings_from)
        lo = 0
        if comm is not None:                                  # this rank's contiguous row-block of the to-matrix (SURVEY.md 8e)
            lo, hi = shard_bounds(len(embeddings_to), comm.world_size, comm.rank)
            y = stage(embeddings_to[lo:hi])
        else:
            y = x if embeddings_to is embeddings_from else stage(embeddings_to)
        # `sparse` thresholds at min_similarity (polyfuzz/models/_utils.py:82); the reference's `sklearn` / `knn` branches
        # ignore it (_utils.py:59-70, 94-102) and blank scores below 0.001 afterwards: threshold 0 here
        if self.cosine_method not in ("sparse", "sklearn", "knn"):
            raise ValueError(f"cosine_method {self.cosine_method!r} unknown (sparse | sklearn | knn)")
        thr = self.min_similarity if self.cosine_method == "sparse" else 0.0
        if exact:                                             # each shard exact; the merge below then equals one GPU
            idx, val, _ = dense.dense_topk_exact(x, y, top_n, thr, self_match=to_list is None, to_index_base=lo)
        else:
            idx, val = dense.dense_topk(x, y, top_n, thr, self_match=to_list is None, to_index_base=lo)
        if comm is not None:
            gi, gv = comm.all_gather_topk(idx.contiguous(), val.contiguous())
            idx, val = merge_topk_any(gi, gv, top_n)
        self.embeddings_to = embeddings_to
        return assemble_matches(from_list, to_list, idx.cpu().numpy(), val.cpu().numpy())
