"""GensimEmbeddings with a FastText model: test infrastructure (no GPU needed).

  ngrams, fnv1a, ngram_ids, subword_vector   a restatement of gensim 4's FastTextKeyedVectors.get_vector for a word outside
                       the vocabulary (DESIGN.md 4.14), written from the rules over characters: the n-grams of "<" + word + ">",
                       32-bit FNV-1a over their UTF-8 bytes sign-extended, bucket = h % bucket, the float32 sum of the rows
                       in list order divided by the count in float32
  FastTextKeyedVectors a stand-in for gensim's class (a KeyedVectorsStandIn, so the reference's isinstance check accepts it)
                       whose get_vector is gensim 4's, over bytes as gensim's compute_ngrams_bytes / ft_hash_bytes walk them:
                       the reference's GensimEmbeddings._embed runs unmodified on it through gensim_oracle.install_gensim
  embed                the restated _embed: every token resolves to a float32 vector when bucket > 0, so every row pools
                       in float32; bucket == 0 is gensim_oracle.embed (unknown tokens are np.zeros, float64 rows)
  edge_vocab           the strings and vocabulary both the CPU and the GPU tests run
  golden_tables        the seeded tables of tests/golden/fasttext_c1.npz, regenerated from the seeds it stores

Parity is pinned to gensim 4's published algorithm and to published test vectors (FNV-1a's, the fastText paper's example), not
to a run of gensim, which these tests do not need."""
import functools

import numpy as np

import gensim_oracle as go


# ---- the restatement ----------------------------------------------------------------------------------------------------------
def ngrams(word, min_n, max_n):
    """The n-grams of "<" + word + ">" as UTF-8 bytes, in gensim's order: start character i ascending, then n = 1..max_n
    ascending while characters remain; kept when n >= min_n and the n-gram is not the lone "<" or ">"."""
    chars = ["<"] + list(word) + [">"]
    out = []
    for i in range(len(chars)):
        for n in range(1, min(max_n, len(chars) - i) + 1):
            if n >= min_n and not (n == 1 and (i == 0 or i == len(chars) - 1)):
                out.append("".join(chars[i:i + n]).encode("utf-8"))
    return out


def fnv1a(data, sign_extend=True):
    """32-bit FNV-1a; gensim and fastText XOR each byte as a signed char widened to 32 bits."""
    h = 2166136261
    for b in data:
        h ^= (b | 0xFFFFFF00) if sign_extend and b >= 0x80 else b
        h = (h * 16777619) & 0xFFFFFFFF
    return h


@functools.lru_cache(maxsize=None)
def _hashes(word, min_n, max_n):
    return np.array([fnv1a(g) for g in ngrams(word, min_n, max_n)], dtype=np.uint64)


def ngram_ids(word, min_n, max_n, bucket):
    return (_hashes(word, min_n, max_n) % np.uint64(bucket)).astype(np.int64)


def _seq_sum32(rows, d):
    """fl32 sequential sum from +0.0 in row order (ufunc.accumulate adds strictly in order; the zero row makes it start from +0.0)."""
    return np.add.accumulate(np.vstack([np.zeros((1, d), np.float32), rows]), axis=0, dtype=np.float32)[-1]


def subword_vector(word, vectors_ngrams, min_n, max_n, bucket):
    """float32 [d]: s = +0.0, s = fl32(s + vectors_ngrams[id]) per n-gram in order, then fl32(s / count); +0.0 without n-grams."""
    d = vectors_ngrams.shape[1]
    ids = ngram_ids(word, min_n, max_n, bucket)
    s = _seq_sum32(vectors_ngrams[ids], d)
    return s if ids.size == 0 else np.divide(s, np.float32(ids.size), dtype=np.float32)


def embed(ft, strings):
    """float64 [n, d]: the reference's np.asarray(_embed(strings), np.float64) on the FastText model `ft`, bit for bit."""
    if ft.bucket == 0:
        return go.embed(ft.key_to_index, ft.vectors, strings)
    V, k2i = np.asarray(ft.vectors), ft.key_to_index
    d = V.shape[1]
    cache = {}
    out = np.empty((len(strings), d), dtype=np.float64)
    for r, s in enumerate(strings):
        toks = s.split(" ")
        rows = []
        for t in toks:
            if t in k2i:
                rows.append(V[k2i[t]])
            else:
                if t not in cache:
                    cache[t] = subword_vector(t, ft.vectors_ngrams, ft.min_n, ft.max_n, ft.bucket)
                rows.append(cache[t])
        # numpy's float32 mean: the sequential float32 sum, divided by the count in float64, rounded to float32
        out[r] = (_seq_sum32(np.stack(rows), d).astype(np.float64) / np.float64(len(toks))).astype(np.float32)
    return out


# ---- gensim 4's FastTextKeyedVectors, as far as get_vector goes ---------------------------------------------------------------
def compute_ngrams_bytes(word, min_n, max_n):
    """gensim/models/fasttext_inner.pyx compute_ngrams_bytes: a walk over the UTF-8 bytes of "<word>"."""
    b = ("<%s>" % word).encode("utf-8")
    out = []
    i = 0
    while i < len(b):
        if b[i] & 0xC0 == 0x80:                                   # not the first byte of a character
            i += 1
            continue
        j, n = i, 1
        while j < len(b) and n <= max_n:
            j += 1
            while j < len(b) and b[j] & 0xC0 == 0x80:
                j += 1
            if n >= min_n and not (n == 1 and (i == 0 or j == len(b))):
                out.append(b[i:j])
            n += 1
        i += 1
    return out


def ft_hash_bytes(data):
    """gensim's ft_hash_bytes: h = h ^ <uint32>(<int8>b); h = h * 16777619, in uint32 arithmetic."""
    h = 2166136261
    for b in data:
        sb = b - 256 if b >= 128 else b                           # <np.int8_t>b
        h = ((h ^ (sb & 0xFFFFFFFF)) * 16777619) & 0xFFFFFFFF      # <np.uint32_t>, then uint32 arithmetic
    return h


def ft_ngram_hashes(word, min_n, max_n, num_buckets):
    return tuple(ft_hash_bytes(g) % num_buckets for g in compute_ngrams_bytes(word, min_n, max_n))


class FastTextKeyedVectors(go.KeyedVectorsStandIn):
    """`vectors`, `vectors_ngrams` [bucket, d], `min_n`, `max_n`, `bucket`, and gensim 4's get_vector (norm=False)."""

    def __init__(self, keys, vectors, vectors_ngrams, min_n, max_n, bucket, key_to_index=None):
        super().__init__(keys, vectors, key_to_index)
        self.vectors_ngrams, self.min_n, self.max_n, self.bucket = vectors_ngrams, min_n, max_n, bucket

    def get_vector(self, word, norm=False):
        if word in self.key_to_index:
            return super().get_vector(word)
        elif self.bucket == 0:
            raise KeyError('cannot calculate vector for OOV word without ngrams')
        else:
            word_vec = np.zeros(self.vectors_ngrams.shape[1], dtype=np.float32)
            ngram_weights = self.vectors_ngrams
            ngram_hashes = ft_ngram_hashes(word, self.min_n, self.max_n, self.bucket)
            if len(ngram_hashes) == 0:
                return word_vec
            for nh in ngram_hashes:
                word_vec += ngram_weights[nh]
            return word_vec / len(ngram_hashes)


# ---- cases ----------------------------------------------------------------------------------------------------------------------
LONG_ASCII = "x" * 2100
LONG_MIXED = "abé中\U0001F600" * 420                       # 2 100 characters of 1-, 2-, 3- and 4-byte UTF-8


def edge_vocab():
    """(keys, strings): ASCII and 2-, 3- and 4-byte UTF-8 tokens, known and unknown; empty tokens and runs of spaces; tokens of
    one character and of 2 100; repeated n-grams ("aaaa"); all-known, all-unknown and mixed rows; and gensim_oracle's cases."""
    keys = ["apple", "house", "a", "é", "中文", "\U0001F600", "similarity", "zz", "aaaa"]
    strings = ["apple", "appl", "appl apple", "aaaa", "aaa", "aaaaa aaaa", "", " ", "   ", "a  b", "b", "é", "été",
               "ÉTÉ é", "中文 中", "中", "\U0001F600", "x\U0001F601y", "\U0001F601", "ÿ", "a b c",
               "apple house zz", "qqq www eee", "apple qqq", " apple", "apple ", "q", "<", ">", "<>", "\t", " x",
               LONG_ASCII, LONG_MIXED, "apple " + LONG_MIXED + " zz", "ࠀ￿\U00010000\U0010FFFF"]
    return keys, strings + go.edge_strings()


def make_model(keys, d, min_n, max_n, bucket, seed=0, vectors_ngrams=None, rows=None):
    """A FastTextKeyedVectors over `keys` with seeded float32 tables (gensim_oracle.random_vectors: +-0.0 sprinkled in, row 0
    all -0.0); `rows` permutes the row each key maps to."""
    V = go.random_vectors(len(keys), d, seed=seed)
    NG = go.random_vectors(max(bucket, 1), d, seed=seed + 1) if vectors_ngrams is None else vectors_ngrams
    k2i = {k: (i if rows is None else int(rows[i])) for i, k in enumerate(keys)}
    if rows is not None:
        Vr = np.empty_like(V); Vr[rows] = V; V = Vr
    return FastTextKeyedVectors(sorted(k2i, key=k2i.get), V, NG[:bucket] if bucket else NG[:0], min_n, max_n, bucket, k2i)


def golden_tables(g):
    """(vectors, vectors_ngrams) of the fixture, regenerated from its seeds."""
    n_rows, d, bucket = len(g["keys"]), int(g["d"]), int(g["bucket"])
    return (go.random_vectors(n_rows, d, seed=int(g["vectors_seed"])),
            go.random_vectors(bucket, d, seed=int(g["ngrams_seed"])))


def golden_model(g):
    V, NG = golden_tables(g)
    k2i = dict(zip(g["keys"].tolist(), g["rows"].tolist()))
    return FastTextKeyedVectors(sorted(k2i, key=k2i.get), V, NG, int(g["min_n"]), int(g["max_n"]), int(g["bucket"]), k2i)
