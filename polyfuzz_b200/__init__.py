"""polyfuzz_b200 -- H100-native (sm_90a) pairwise string-similarity hot path behind PolyFuzz's
BaseMatcher plugin API.  See DESIGN.md / INTEGRATION.md."""
from .matchers import BaseMatcher, TFIDF, RapidFuzz, EditDistance, Embeddings, GensimEmbeddings  # noqa: F401
from .linkage import single_linkage, install_linkage  # noqa: F401

__version__ = "0.1.0"


def install():
    """Make the reference's string shortcuts -- PolyFuzz("TF-IDF"), PolyFuzz("EditDistance"), PolyFuzz("Embeddings")
    (polyfuzz/polyfuzz.py:124-133) -- construct this package's matchers: the names the unmodified orchestrator looks up in its own
    module (and polyfuzz.models) are rebound to the classes of this package.  No reference source is modified."""
    import polyfuzz.models as pm
    import polyfuzz.polyfuzz as pp
    for name, cls in (("TFIDF", TFIDF), ("RapidFuzz", RapidFuzz), ("EditDistance", EditDistance), ("Embeddings", Embeddings)):
        for mod in (pp, pm):
            if hasattr(mod, name):
                setattr(mod, name, cls)
