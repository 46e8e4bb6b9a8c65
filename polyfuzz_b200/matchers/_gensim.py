"""GensimEmbeddings matcher -- drop-in for polyfuzz.models.GensimEmbeddings (polyfuzz/models/_gensim.py): each string is the
mean of its space-split tokens' word vectors, pooled on the device (K6, DESIGN.md 4.11) bit for bit as the reference's `_embed`
does, then matched by Embeddings.match unchanged (K4, either precision, any top_n, distributed or not).

The model is a gensim KeyedVectors, or any object with `key_to_index`, `index_to_key` and a 2-D `vectors` array (gensim is not
a dependency); a string is loaded with gensim.downloader.load as the reference does.  The vocabulary goes to the device on the
first match, so constructing the matcher needs no GPU.

A FastText model (gensim's FastTextKeyedVectors) also carries `vectors_ngrams` [bucket, d], `min_n`, `max_n` and `bucket`; its
get_vector builds a word outside the vocabulary from the rows of its character n-grams, and so does the device (K6's
pfz_ft_pool, DESIGN.md 4.14), bit for bit.  Both tables must be float32, as gensim makes them.  A string list holding a
surrogate code point raises UnicodeEncodeError, as the reference's str.encode("utf-8") does for an unknown word; the check
covers every string, so it also raises when every surrogate-bearing token is a vocabulary key, where the reference does not.
A FastText-looking model without that subword surface is refused with NotImplementedError."""
import numpy as np
import torch

from ._embeddings import Embeddings
from .. import wordvec

_MODEL_ERROR = ("Please select a correct Gensim model: \n"
                "`import gensim.downloader as api` \n"
                "`ft = api.load('fasttext-wiki-news-subwords-300')`")


def _is_fasttext(model):
    return hasattr(model, "buckets_word") or any(c.__name__ == "FastTextKeyedVectors" for c in type(model).__mro__)


def _has_subwords(model):
    return all(hasattr(model, a) for a in ("vectors_ngrams", "min_n", "max_n", "bucket")) and np.ndim(model.vectors_ngrams) == 2


def _is_keyed_vectors(model):
    return all(hasattr(model, a) for a in ("key_to_index", "index_to_key", "vectors")) and np.ndim(model.vectors) == 2


class GensimEmbeddings(Embeddings):
    def __init__(self, embedding_model="fasttext-wiki-news-subwords-300", min_similarity: float = 0.75, top_n: int = 1,
                 cosine_method: str = "sparse", model_id: str = None, distributed: bool = False, precision: str = "bf16"):
        super().__init__(None, min_similarity, top_n, cosine_method, model_id, distributed, precision)
        if isinstance(embedding_model, str):
            import gensim.downloader as api                 # ModuleNotFoundError without gensim, as in the reference
            embedding_model = api.load(embedding_model)
        fasttext = _is_fasttext(embedding_model)
        if fasttext and not _has_subwords(embedding_model):
            raise NotImplementedError("FastText models need vectors_ngrams, min_n, max_n and bucket to build vectors for "
                                      "unknown words from character n-grams: pass a gensim 4 FastTextKeyedVectors or a KeyedVectors model")
        if not _is_keyed_vectors(embedding_model):
            raise ValueError(_MODEL_ERROR)
        wordvec.check_vectors(embedding_model.vectors, len(embedding_model.key_to_index))
        if fasttext:
            m = embedding_model
            wordvec.check_subwords(m.vectors, m.vectors_ngrams, m.min_n, m.max_n, m.bucket)
        self.embedding_model = embedding_model
        self._wv = None                                     # the device vocabulary (wordvec.WordVectors), built on first use

    def _embed(self, strings):
        """float64 [n, d] device tensor, equal to the reference's _embed(strings) bit for bit."""
        if self._wv is None:
            m = self.embedding_model
            sub = dict(vectors_ngrams=m.vectors_ngrams, min_n=m.min_n, max_n=m.max_n, bucket=m.bucket) if _is_fasttext(m) else {}
            self._wv = wordvec.WordVectors(m.key_to_index, m.vectors, **sub)
        return self._wv.pool(strings)

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_wv"] = None
        if isinstance(st.get("embeddings_to"), torch.Tensor):
            st["embeddings_to"] = st["embeddings_to"].cpu().numpy()
        return st
