"""GPU matchers: BaseMatcher plugins for PolyFuzz (see ../../INTEGRATION.md)."""
from ._base import BaseMatcher, register_with_reference  # noqa: F401
from ._embeddings import Embeddings  # noqa: F401
from ._gensim import GensimEmbeddings  # noqa: F401
from ._rapidfuzz import EditDistance, RapidFuzz  # noqa: F401
from ._tfidf import TFIDF  # noqa: F401

__all__ = ["BaseMatcher", "TFIDF", "RapidFuzz", "EditDistance", "Embeddings", "GensimEmbeddings"]
