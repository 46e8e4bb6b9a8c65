"""GensimEmbeddings test infrastructure (no GPU needed).

  KeyedVectorsStandIn  the lookup surface of gensim's KeyedVectors that the reference's GensimEmbeddings uses
  install_gensim       the reference's import shim plus, where gensim is absent, a stub gensim.models.keyedvectors whose
                       Word2VecKeyedVectors is the stand-in, so polyfuzz/models/_gensim.py runs unmodified
  embed                a numpy restatement of the reference's _embed (polyfuzz/models/_gensim.py:118-140), written as explicit
                       loops in the order numpy adds (DESIGN.md 4.11)
  edge_cases           the strings and vocabularies both the CPU and the GPU tests run"""
import sys
import types

import numpy as np


class KeyedVectorsStandIn:
    """`vectors` [n, d], `index_to_key`, `key_to_index`, and get_index / get_vector with gensim's semantics
    (vectors[key_to_index[key]], else KeyError).  key_to_index defaults to each key's position in `keys`."""

    def __init__(self, keys, vectors, key_to_index=None):
        self.vectors = vectors
        self.index_to_key = list(keys)
        self.key_to_index = dict(key_to_index) if key_to_index is not None else {k: i for i, k in enumerate(self.index_to_key)}

    def get_index(self, key):
        val = self.key_to_index.get(key, -1)
        if val >= 0:
            return val
        raise KeyError(f"Key '{key}' not present")

    def get_vector(self, key):
        return self.vectors[self.get_index(key)]


def install_gensim(reference_root=None) -> bool:
    """ref_shim.install(), and where gensim is absent a stub `gensim.models.keyedvectors` (Word2VecKeyedVectors =
    KeyedVectorsStandIn).  `gensim` stays a plain module, so `import gensim.downloader` still raises ModuleNotFoundError.
    Returns False when a real gensim is installed: nothing is stubbed, and the stand-in is not the reference's model type."""
    from oracle import ref_shim
    if reference_root is not None:
        ref_shim.REFERENCE_ROOT = reference_root
    ref_shim.install()
    mod = sys.modules.get("gensim.models.keyedvectors")
    if mod is not None:
        return getattr(mod, "Word2VecKeyedVectors", None) is KeyedVectorsStandIn
    try:
        import gensim  # noqa: F401
        return False
    except ModuleNotFoundError:
        pass
    kv = types.ModuleType("gensim.models.keyedvectors")
    kv.Word2VecKeyedVectors = kv.KeyedVectors = KeyedVectorsStandIn
    models = types.ModuleType("gensim.models")
    models.keyedvectors = kv
    gensim = types.ModuleType("gensim")
    gensim.models = models
    sys.modules.update({"gensim": gensim, "gensim.models": models, "gensim.models.keyedvectors": kv})
    return True


def embed(key_to_index, vectors, strings):
    """float64 [n, d]: the reference's np.asarray(_embed(strings), np.float64), bit for bit.
    Tokens: s.split(" ").  A row whose tokens are all keys of a float32 table is summed in float32 (from +0.0, one rounded
    add per token: numpy's add.reduce starts from its identity, so a sum of -0.0 values is +0.0), and numpy's mean divides that
    sum by the token count in float64 and rounds to float32.  Any other row is float64 throughout, summed the same way from
    +0.0; missing tokens are +0.0 (np.zeros(d))."""
    V = np.asarray(vectors)
    d = V.shape[1]
    out = np.empty((len(strings), d), dtype=np.float64)
    for r, s in enumerate(strings):
        rows = [key_to_index.get(t) for t in s.split(" ")]
        n = len(rows)
        if V.dtype == np.float32 and all(x is not None for x in rows):
            acc = np.zeros(d, dtype=np.float32)
            for x in rows:
                acc = np.add(acc, V[x], dtype=np.float32)
            out[r] = (acc.astype(np.float64) / np.float64(n)).astype(np.float32)
        else:
            acc = np.zeros(d, dtype=np.float64)
            for x in rows:
                acc = np.add(acc, np.zeros(d) if x is None else V[x].astype(np.float64), dtype=np.float64)
            out[r] = acc / np.float64(n)
    return out


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def random_vectors(n, d, seed, dtype=np.float32):
    """Seeded vectors with exact zeros of both signs sprinkled in, so that the sign of a zero sum is exercised."""
    rng = np.random.default_rng(seed)
    V = rng.standard_normal((n, d)).astype(dtype)
    z = rng.random((n, d))
    V[z < 0.05] = 0.0
    V[z > 0.95] = -0.0
    if n:
        V[0] = -0.0                                       # a key whose vector is all -0.0
    return V


EDGE_KEYS = ["apple", "apples", "appl", "app", "a", "b", "mouse", "house", "similarity", "recal", "", "ap", "appla",
             "tab\there", "nb sp", "\U0001F600", "\U0001F600x", "x\U0001F601", "été", "ÉTÉ", "zz"]


def edge_strings():
    """Strings for the restatement and the device: the README lists, empty and space-only strings, runs of spaces, tabs, NBSP,
    tokens beyond the BMP, all-missing, all-found and mixed rows, and strings of thousands of tokens."""
    base = ["apple", "apples", "appl", "recal", "house", "similarity", "apple", "apples", "mouse",
            "", " ", "  ", "  a  b ", "a b", "b a", "apple apple apple", "tab\there apple", "tab here", "nb sp b",
            "nb sp", "\U0001F600 \U0001F600x x\U0001F601", "\U0001F600x\U0001F600", "été ÉTÉ", "qqq www",
            "qqq", "apple qqq", " apple", "apple ", "ap appla app", "appl apple", "zz", "zz zz zz zz zz zz zz zz zz"]
    rng = np.random.default_rng(7)
    words = EDGE_KEYS + ["oov1", "oov2", "中文"]
    long = [" ".join(rng.choice(words, size=n)) for n in (31, 32, 33, 257, 3000)]
    long.append(" ".join(["apple"] * 4000))                 # all found, one key
    long.append(" ".join(["nope"] * 2500))                  # all missing
    long.append(" " * 1500)                                 # 1501 empty tokens
    return base + long


def prefix_vocab():
    """A vocabulary whose keys include "", keys that are prefixes of each other and keys differing only in their last code
    point, with strings that look each of them up and near misses."""
    stems = ["", "a", "ab", "abc", "abcd", "abcde", "é", "éé", "\U0001F600", "\U0001F600\U0001F600"]
    keys = list(stems)
    for s in ["k", "ke", "key", "中"]:
        keys += [s + chr(c) for c in range(0x61, 0x61 + 12)] + [s + chr(0x10000 + c) for c in range(4)]
    strings = [" ".join(keys[i:i + 5]) for i in range(0, len(keys), 3)]
    strings += ["abcdef", "abcd abcdf", "kz key{ \U0001F600\U0001F600\U0001F600", " ", "", "a  ab   abc", "ééé é"]
    return keys, strings
