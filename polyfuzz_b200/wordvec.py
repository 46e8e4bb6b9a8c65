"""K6 host driver: word-vector lookup and mean pooling on the device (include/pfz.h, pfz_wv_*), the embedding step of
GensimEmbeddings (polyfuzz/models/_gensim.py:118-140).  The vocabulary is staged once (key code points, each key's row, the
vectors and a hash table over the keys); pooling a string list is then one H2D copy of the strings and four launches (count,
scan, lookup, pool), with no host synchronisation, into a float64 [n, d] tensor bit-identical to the reference's matrix.

For a FastText model (gensim's FastTextKeyedVectors, DESIGN.md 4.14) the subword table `vectors_ngrams` [bucket, d] is staged
too, and when bucket > 0 the pool launch is pfz_ft_pool: a token outside the vocabulary gets the mean of its character
n-grams' rows, as get_vector does, instead of a zero vector."""
import numpy as np
import torch

from . import _lib
from .engine import _dev, _p, _stream, _to_dev, _ws
from .strings import pack_strings


def check_vectors(vectors, n_keys):
    """The vector table the device pools from: 2-D, float32 or float64, d >= 2, and at least one key.  Raises ValueError."""
    V = np.asarray(vectors)
    if V.ndim != 2:
        raise ValueError(f"the word vectors must be a 2-D array [n_keys, d], got shape {V.shape}")
    if V.dtype not in (np.float32, np.float64):
        raise ValueError(f"word vectors of dtype {V.dtype} are not supported (float32 or float64)")
    if V.shape[1] < 2:
        # for d = 1 numpy's axis-0 mean sums pairwise once a string has 8 tokens or more, not in token order
        raise ValueError("word vectors of dimension 1 are not supported (d >= 2)")
    if n_keys == 0 or V.shape[0] == 0:
        raise ValueError("the word-vector vocabulary is empty")
    return V


def check_subwords(vectors, vectors_ngrams, min_n, max_n, bucket):
    """The subword surface of a FastText model: float32 `vectors` and `vectors_ngrams` of one width, at least `bucket` rows of
    n-grams, 0 <= bucket < 2^32 and 0 <= min_n, max_n < 2^31.  Raises ValueError; returns vectors_ngrams as an array."""
    V, NG = np.asarray(vectors), np.asarray(vectors_ngrams)
    if NG.ndim != 2:
        raise ValueError(f"vectors_ngrams must be a 2-D array [bucket, d], got shape {NG.shape}")
    if V.dtype != np.float32 or NG.dtype != np.float32:
        # gensim keeps both in float32; get_vector adds n-gram rows in place into a float32 vector
        raise ValueError(f"FastText vectors ({V.dtype}) and vectors_ngrams ({NG.dtype}) must both be float32")
    if NG.shape[1] != V.shape[1]:
        raise ValueError(f"vectors_ngrams has width {NG.shape[1]}, the vectors {V.shape[1]}")
    for name, v in (("bucket", bucket), ("min_n", min_n), ("max_n", max_n)):
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
            raise ValueError(f"{name} must be an integer, got {v!r}")
    if not 0 <= bucket < 1 << 32:
        raise ValueError(f"bucket {bucket} must be in [0, 2^32)")
    if NG.shape[0] < bucket:
        raise ValueError(f"vectors_ngrams has {NG.shape[0]} rows, fewer than bucket ({bucket})")
    if not (0 <= min_n < 1 << 31 and 0 <= max_n < 1 << 31):
        raise ValueError(f"min_n ({min_n}) and max_n ({max_n}) must be in [0, 2^31)")
    return NG


def check_no_surrogates(blob, off, strings):
    """UnicodeEncodeError for the first string holding a surrogate code point, as str.encode("utf-8") raises it."""
    if blob.dtype != np.uint32:
        return
    bad = np.flatnonzero((blob >= 0xD800) & (blob <= 0xDFFF))
    if bad.size:
        r = int(np.searchsorted(off, bad[0], side="right")) - 1
        p = int(bad[0] - off[r])
        raise UnicodeEncodeError("utf-8", strings[r], p, p + 1, "surrogates not allowed")


def _blob_to_dev(blob):
    """Packed code points (uint8 for an ASCII list, else uint32) -> int32 device tensor of at least one element."""
    if blob.size == 0:
        return torch.zeros(1, dtype=torch.int32, device=_dev())
    if blob.dtype == np.uint8:
        return _to_dev(blob).to(torch.int32)
    return _to_dev(blob.view(np.int32), torch.int32)


def default_cap(n_keys):
    """The table size used unless one is given: the smallest power of two >= 2 * n_keys (load factor at most 1/2)."""
    return 1 << max(1, int(2 * n_keys - 1).bit_length())


class WordVectors:
    """A KeyedVectors vocabulary resident on the device.  key_to_index: {str: row of `vectors`}; cap: hash-table slots (a power
    of two above the number of keys; default_cap by default).  A FastText model also passes vectors_ngrams, min_n, max_n and
    bucket (check_subwords); with bucket > 0 the subword table is staged and unknown tokens get subword vectors."""

    def __init__(self, key_to_index, vectors, cap=None, vectors_ngrams=None, min_n=0, max_n=0, bucket=0):
        keys = list(key_to_index)
        V = check_vectors(vectors, len(keys))
        NG = None if vectors_ngrams is None else check_subwords(V, vectors_ngrams, min_n, max_n, bucket)
        rows = np.fromiter((key_to_index[k] for k in keys), dtype=np.int64, count=len(keys))
        if rows.min() < 0 or rows.max() >= V.shape[0]:
            raise ValueError("key_to_index maps a key outside the rows of the vectors")
        cap = default_cap(len(keys)) if cap is None else int(cap)
        if cap & (cap - 1) or cap <= len(keys) or cap > 1 << 31:
            raise ValueError(f"cap {cap} must be a power of two above the number of keys ({len(keys)}), at most 2^31")
        self.n_keys, self.d, self.cap = len(keys), int(V.shape[1]), cap
        self.bucket, self.min_n, self.max_n = (int(bucket), int(min_n), int(max_n)) if NG is not None else (0, 0, 0)
        blob, off, _ = pack_strings(keys)                  # TypeError for a key that is not str
        self.key_blob, self.key_off = _blob_to_dev(blob), _to_dev(off)
        self.key_row = _to_dev(rows.astype(np.int32))
        self.vectors = torch.from_numpy(np.ascontiguousarray(V)).to(_dev())
        self.table = torch.empty(cap, dtype=torch.int32, device=_dev())
        _lib.call("pfz_wv_table_build", _p(self.key_blob), _p(self.key_off), self.n_keys, _p(self.table), cap, _stream())
        # the subword table (bucket * d * 4 bytes: 2.4 GB at 2M x 300), only where unknown tokens read it
        self.vectors_ngrams = torch.from_numpy(np.ascontiguousarray(NG[:self.bucket])).to(_dev()) if self.bucket else None

    def _lookup(self, strings):
        strings = strings if isinstance(strings, (list, tuple)) else list(strings)
        n = len(strings)
        if n >= 1 << 31:
            raise ValueError("at most 2^31 - 1 strings per call")
        dev = _dev()
        blob, off, _ = pack_strings(strings)
        if self.bucket:
            check_no_surrogates(blob, off, strings)                 # before any device work
        tok_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
        tok_row = torch.empty(max(int(off[-1]) + n, 1), dtype=torch.int32, device=dev)   # tokens <= spaces + n <= code points + n
        if n == 0:
            tok_off.zero_()
            return tok_off, tok_row[:0], None, None
        ws_bytes = int(_lib.load().pfz_wv_lookup_ws_bytes(n))
        # held until the launches are enqueued: a tensor freed earlier could hand its memory to the next allocation
        d_blob, d_off, ws = _blob_to_dev(blob), _to_dev(off), _ws(ws_bytes)
        _lib.call("pfz_wv_lookup", _p(d_blob), _p(d_off), n, _p(self.key_blob), _p(self.key_off), _p(self.key_row),
                  _p(self.table), self.cap, _p(tok_off), _p(tok_row), _p(ws), ws_bytes, _stream())
        return tok_off, tok_row, d_blob, d_off

    def lookup(self, strings):
        """(tok_off int64[n+1], tok_row int32) on the device: each string's tokens and their rows of V (-1 = missing)."""
        return self._lookup(strings)[:2]

    def pool(self, strings):
        """float64 [n, d] device tensor: row i = the reference's _embed row of strings[i], bit for bit."""
        tok_off, tok_row, d_blob, d_off = self._lookup(strings)
        n = tok_off.numel() - 1
        out = torch.empty((n, self.d), dtype=torch.float64, device=_dev())
        if self.bucket and n:
            _lib.call("pfz_ft_pool", _p(d_blob), _p(d_off), n, _p(tok_off), _p(tok_row), _p(self.vectors), _p(self.vectors_ngrams),
                      self.d, self.bucket, self.min_n, self.max_n, _p(out), self.d, _stream())
        else:
            _lib.call("pfz_wv_pool", _p(self.vectors), int(self.vectors.dtype == torch.float64), self.d, _p(tok_off), _p(tok_row), n,
                      _p(out), self.d, _stream())
        return out
