"""GensimEmbeddings matcher -- drop-in for polyfuzz.models.GensimEmbeddings (polyfuzz/models/_gensim.py): each string is the
mean of its space-split tokens' word vectors, pooled on the device (K6, DESIGN.md 4.11) bit for bit as the reference's `_embed`
does, then matched by Embeddings.match unchanged (K4, either precision, any top_n, distributed or not).

The model is a gensim KeyedVectors, or any object with `key_to_index`, `index_to_key` and a 2-D `vectors` array (gensim is not
a dependency); a string is loaded with gensim.downloader.load as the reference does.  FastText models, which build vectors for
unknown words from character n-grams, are refused.  The vocabulary goes to the device on the first match, so constructing the
matcher needs no GPU."""
import numpy as np
import torch

from ._embeddings import Embeddings
from .. import wordvec

_MODEL_ERROR = ("Please select a correct Gensim model: \n"
                "`import gensim.downloader as api` \n"
                "`ft = api.load('fasttext-wiki-news-subwords-300')`")


def _is_fasttext(model):
    return hasattr(model, "buckets_word") or any(c.__name__ == "FastTextKeyedVectors" for c in type(model).__mro__)


def _is_keyed_vectors(model):
    return all(hasattr(model, a) for a in ("key_to_index", "index_to_key", "vectors")) and np.ndim(model.vectors) == 2


class GensimEmbeddings(Embeddings):
    def __init__(self, embedding_model="fasttext-wiki-news-subwords-300", min_similarity: float = 0.75, top_n: int = 1,
                 cosine_method: str = "sparse", model_id: str = None, distributed: bool = False, precision: str = "bf16"):
        super().__init__(None, min_similarity, top_n, cosine_method, model_id, distributed, precision)
        if isinstance(embedding_model, str):
            import gensim.downloader as api                 # ModuleNotFoundError without gensim, as in the reference
            embedding_model = api.load(embedding_model)
        if _is_fasttext(embedding_model):
            raise NotImplementedError("FastText models build vectors for unknown words from character n-grams, which is not "
                                      "supported: pass a KeyedVectors model")
        if not _is_keyed_vectors(embedding_model):
            raise ValueError(_MODEL_ERROR)
        wordvec.check_vectors(embedding_model.vectors, len(embedding_model.key_to_index))
        self.embedding_model = embedding_model
        self._wv = None                                     # the device vocabulary (wordvec.WordVectors), built on first use

    def _embed(self, strings):
        """float64 [n, d] device tensor, equal to the reference's _embed(strings) bit for bit."""
        if self._wv is None:
            self._wv = wordvec.WordVectors(self.embedding_model.key_to_index, self.embedding_model.vectors)
        return self._wv.pool(strings)

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_wv"] = None
        if isinstance(st.get("embeddings_to"), torch.Tensor):
            st["embeddings_to"] = st["embeddings_to"].cpu().numpy()
        return st
