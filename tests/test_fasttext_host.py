"""GensimEmbeddings with a FastText model, without a GPU: the restatement of gensim 4's subword vectors (tests/fasttext_oracle.py)
against published answers, against the reference's _embed on the gensim stand-in and against the golden fixture, bit for bit;
and the matcher's host checks."""
import os
import pickle

import numpy as np
import pytest

import fasttext_oracle as fo
import gensim_oracle as go
from oracle import ref_shim

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fasttext_c1.npz")
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="the reference is not present")
MIN_MAX = [(3, 6), (1, 1), (1, 3), (2, 2), (0, 2), (4, 3), (5, 40)]


@pytest.fixture(scope="module")
def RefGensim():
    if not go.install_gensim():
        pytest.skip("a real gensim is installed: the reference needs its own KeyedVectors there")
    from polyfuzz.models._gensim import GensimEmbeddings
    return GensimEmbeddings


def _golden():
    z = np.load(GOLDEN)
    return {k: z[k] for k in z.files}


# ---- published answers ------------------------------------------------------------------------------------------------------------
def test_fnv1a_published_vectors():
    assert [fo.fnv1a(s) for s in (b"", b"a", b"foobar")] == [0x811C9DC5, 0xE40C292C, 0xBF9CF968]
    assert [fo.ft_hash_bytes(s) for s in (b"", b"a", b"foobar")] == [0x811C9DC5, 0xE40C292C, 0xBF9CF968]


def test_ngram_known_answers():
    assert fo.ngrams("where", 3, 3) == [b"<wh", b"whe", b"her", b"ere", b"re>"]            # the fastText paper's example
    assert fo.ngrams("ab", 1, 3) == [b"<a", b"<ab", b"a", b"ab", b"ab>", b"b", b"b>"]
    assert fo.ngrams("", 1, 6) == [b"<>"] and fo.ngrams("", 3, 6) == []
    e = "é".encode("utf-8")
    assert fo.ngrams("é", 1, 2) == [b"<" + e, e, e + b">"]
    assert fo.fnv1a(e) == 0x3CFA68C1 and fo.fnv1a(e, sign_extend=False) == 0x1E9DE8C1   # tells the two byte rules apart
    assert fo.ft_hash_bytes(e) == 0x3CFA68C1


def test_ngrams_and_hashes_equal_gensims_byte_walk():
    _, strings = fo.edge_vocab()
    words = sorted({t for s in strings for t in s.split(" ")})
    for mn, mx in MIN_MAX:
        for w in words:
            assert fo.ngrams(w, mn, mx) == fo.compute_ngrams_bytes(w, mn, mx), (w, mn, mx)
    for g in fo.ngrams(fo.LONG_MIXED[:40], 1, 6) + fo.ngrams("ࠀ￿\U00010000\U0010FFFF", 1, 4):
        assert fo.fnv1a(g) == fo.ft_hash_bytes(g)


def test_subword_vector_rules():
    NG = go.random_vectors(7, 3, seed=1)
    assert fo.subword_vector("", NG, 3, 6, 7).tobytes() == np.zeros(3, np.float32).tobytes()          # no n-grams: +0.0
    NG0 = np.full((1, 3), -0.0, np.float32)
    assert fo.subword_vector("ab", NG0, 1, 3, 1).tobytes() == np.zeros(3, np.float32).tobytes()      # sum from +0.0
    v = fo.subword_vector("aaaa", NG, 1, 2, 7)
    ids = fo.ngram_ids("aaaa", 1, 2, 7)
    assert len(ids) == 9 and len(set(ids.tolist())) < 9                # duplicates stay in the list
    s = np.zeros(3, np.float32)
    for i in ids:
        s = np.float32(s + NG[i])
    assert v.tobytes() == (s / np.float32(9)).astype(np.float32).tobytes()


# ---- the restatement against the reference ------------------------------------------------------------------------------------------
def _ref_embed(RefGensim, ft, strings):
    out = RefGensim(ft)._embed(strings)
    return np.asarray(out, np.float64)


@needs_ref
@pytest.mark.parametrize("min_n,max_n", MIN_MAX)
@pytest.mark.parametrize("bucket", [1, 7, 2003])
def test_restatement_equals_reference_embed(RefGensim, min_n, max_n, bucket):
    keys, strings = fo.edge_vocab()
    if (min_n, max_n) == (5, 40):
        strings = [s for s in strings if len(s) < 3000]            # the long tokens run in the GPU tests
    ft = fo.make_model(keys, 31, min_n, max_n, bucket, seed=bucket, rows=np.random.default_rng(bucket).permutation(len(keys)))
    got = fo.embed(ft, strings)
    ref = _ref_embed(RefGensim, ft, strings)
    assert np.array_equal(go.bits(got), go.bits(ref))
    assert RefGensim(ft)._embed(["qqq"]).dtype == np.float32       # unknown tokens keep the row on the float32 path


@needs_ref
@pytest.mark.parametrize("d", [2, 32, 33, 300])
def test_restatement_equals_reference_embed_across_widths(RefGensim, d):
    keys, strings = fo.edge_vocab()
    strings = [s for s in strings if len(s) < 3000]
    ft = fo.make_model(keys, d, 3, 6, 7, seed=d)
    assert np.array_equal(go.bits(fo.embed(ft, strings)), go.bits(_ref_embed(RefGensim, ft, strings)))


@needs_ref
def test_bucket_zero_is_the_keyed_vectors_result(RefGensim):
    keys, strings = fo.edge_vocab()
    strings = strings[:40]
    ft = fo.make_model(keys, 33, 3, 6, 0, seed=3)
    ref = RefGensim(ft)._embed(strings)
    assert ref.dtype == np.float64                                 # unknown tokens are np.zeros: float64 rows
    assert np.array_equal(go.bits(fo.embed(ft, strings)), go.bits(ref))
    assert np.array_equal(go.bits(go.embed(ft.key_to_index, ft.vectors, strings)), go.bits(ref))


@needs_ref
def test_restatement_equals_reference_on_the_golden_model(RefGensim):
    g = _golden()
    ft = fo.golden_model(g)
    strings = g["strings"].tolist()
    assert np.array_equal(go.bits(_ref_embed(RefGensim, ft, strings)), go.bits(fo.embed(ft, strings)))


def test_restatement_equals_golden_embed():
    g = _golden()
    ft = fo.golden_model(g)
    strings = g["strings"].tolist()
    assert any(not s.isascii() for s in strings)
    assert any(t not in ft.key_to_index for s in strings for t in s.split(" "))
    assert np.array_equal(go.bits(fo.embed(ft, strings)), go.bits(g["embed"]))


# ---- the matcher's host logic ---------------------------------------------------------------------------------------------------
def _ft(**kw):
    a = dict(keys=["w0", "w1", "w2"], d=4, min_n=3, max_n=6, bucket=11)
    a.update(kw)
    return fo.make_model(a["keys"], a["d"], a["min_n"], a["max_n"], a["bucket"])


def test_constructor_accepts_fasttext_models():
    from polyfuzz_b200 import GensimEmbeddings
    for kw in ({}, dict(bucket=0), dict(min_n=0, max_n=0), dict(min_n=5, max_n=3), dict(bucket=(1 << 32) - 1)):
        ft = _ft(**kw) if kw.get("bucket") != (1 << 32) - 1 else None
        if ft is None:                                              # bucket near 2^32 over a view with that many rows
            ft = _ft(bucket=1)
            ft.bucket = (1 << 32) - 1
            ft.vectors_ngrams = np.lib.stride_tricks.as_strided(ft.vectors_ngrams, shape=(ft.bucket, 4), strides=(0, 4))
        m = GensimEmbeddings(ft, min_similarity=0.5, top_n=3, precision="fp64")
        assert m._wv is None and m.embedding_model is ft and (m.top_n, m.precision) == (3, "fp64")


def test_constructor_refusals():
    from polyfuzz_b200 import GensimEmbeddings
    cases = [
        (dict(vectors=lambda f: f.vectors.astype(np.float64)), "float32"),
        (dict(vectors_ngrams=lambda f: f.vectors_ngrams.astype(np.float64)), "float32"),
        (dict(vectors_ngrams=lambda f: f.vectors_ngrams.astype(np.float16)), "float32"),
        (dict(vectors_ngrams=lambda f: np.ones((11, 5), np.float32)), "width"),
        (dict(vectors_ngrams=lambda f: f.vectors_ngrams[:10]), "fewer than bucket"),
        (dict(bucket=lambda f: 1 << 32), r"2\^32"),
        (dict(bucket=lambda f: -1), r"2\^32"),
        (dict(min_n=lambda f: -1), "min_n"),
        (dict(max_n=lambda f: -2), "max_n"),
        (dict(max_n=lambda f: 6.0), "integer"),
    ]
    for change, msg in cases:
        ft = _ft()
        for k, fn in change.items():
            setattr(ft, k, fn(ft))
        with pytest.raises(ValueError, match=msg):
            GensimEmbeddings(ft)
    # a FastText model without the subword surface is still refused
    ft = _ft()
    del ft.bucket
    with pytest.raises(NotImplementedError, match="FastText"):
        GensimEmbeddings(ft)
    ft = _ft()
    ft.vectors_ngrams = np.ones(4, np.float32)
    with pytest.raises(NotImplementedError, match="FastText"):
        GensimEmbeddings(ft)
    with pytest.raises(ValueError, match="dimension 1"):
        GensimEmbeddings(_ft(d=1))
    with pytest.raises(ValueError, match="empty"):
        GensimEmbeddings(_ft(keys=[]))


def test_surrogates_raise_unicode_encode_error_before_device_work():
    from polyfuzz_b200 import wordvec
    from polyfuzz_b200.strings import pack_strings
    for strings in (["apple"], ["é 中"], ["a\U0001F600"]):
        blob, off, _ = pack_strings(strings)
        wordvec.check_no_surrogates(blob, off, strings)
    strings = ["apple", "é", "ab c\ud800d", "\udfff"]
    blob, off, _ = pack_strings(strings)
    with pytest.raises(UnicodeEncodeError) as e:
        wordvec.check_no_surrogates(blob, off, strings)
    assert (e.value.object, e.value.start, e.value.end) == ("ab c\ud800d", 4, 5)
    with pytest.raises(UnicodeEncodeError):                         # what the reference meets for an unknown word
        ("<%s>" % "c\ud800d").encode("utf-8")


def test_pickle_drops_the_device_tables():
    from polyfuzz_b200 import GensimEmbeddings
    m = GensimEmbeddings(_ft(), top_n=2)
    m._wv = object()
    st = pickle.loads(pickle.dumps(m))
    assert st._wv is None and st.embedding_model.bucket == 11 and type(st.embedding_model).__name__ == "FastTextKeyedVectors"
    assert np.array_equal(st.embedding_model.vectors_ngrams, m.embedding_model.vectors_ngrams)
