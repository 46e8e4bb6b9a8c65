"""GensimEmbeddings without a GPU: the numpy restatement of the reference's _embed (tests/gensim_oracle.py) against the
reference itself and the golden fixture, bit for bit, and the matcher's host logic (constructor validation, pickling)."""
import os
import pickle

import numpy as np
import pytest
import torch

import gensim_oracle as go
from oracle import ref_shim

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gensim_c1.npz")
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="the reference is not present")


@pytest.fixture(scope="module")
def RefGensim():
    if not go.install_gensim():
        pytest.skip("a real gensim is installed: the reference needs its own KeyedVectors there")
    from polyfuzz.models._gensim import GensimEmbeddings
    return GensimEmbeddings


def _golden():
    z = np.load(GOLDEN)
    return {k: z[k] for k in z.files}


def _ref_embed(RefGensim, keys, V, strings, k2i=None):
    kv = go.KeyedVectorsStandIn(keys, V, k2i)
    return np.asarray(RefGensim(kv)._embed(strings), np.float64)


def _edge_vocab(with_empty):
    keys = [k for k in go.EDGE_KEYS if with_empty or k != ""]
    return [k for k in keys if k not in ("mouse", "zz")] + ["zz"]      # "mouse" missing, "zz" found


@needs_ref
@pytest.mark.parametrize("d", [2, 25, 31, 32, 33, 300])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("with_empty", [False, True])
def test_restatement_equals_reference_on_edge_cases(RefGensim, d, dtype, with_empty):
    keys = _edge_vocab(with_empty)
    V = go.random_vectors(len(keys), d, seed=d, dtype=dtype)
    strings = go.edge_strings()
    k2i = {k: i for i, k in enumerate(keys)}
    got = go.embed(k2i, V, strings)
    assert np.array_equal(go.bits(got), go.bits(_ref_embed(RefGensim, keys, V, strings)))
    # the rows took the paths the test means to cover: float32 and float64 sums, and -0.0 inputs (which pool to +0.0)
    found = [all(t in k2i for t in s.split(" ")) for s in strings]
    assert any(found) and not all(found)
    assert (go.bits(V.astype(np.float64)) == np.uint64(1 << 63)).any() and (go.bits(got) == 0).any()


@needs_ref
def test_restatement_equals_reference_on_prefix_vocab(RefGensim):
    keys, strings = go.prefix_vocab()
    V = go.random_vectors(len(keys), 33, seed=5)
    rows = np.random.default_rng(3).permutation(len(keys))
    k2i = {k: int(r) for k, r in zip(keys, rows)}
    Vr = np.empty_like(V); Vr[rows] = V
    got = go.embed(k2i, Vr, strings)
    assert np.array_equal(go.bits(got), go.bits(_ref_embed(RefGensim, sorted(k2i, key=k2i.get), Vr, strings, k2i)))


@needs_ref
def test_restatement_equals_reference_on_the_golden_vocabularies(RefGensim):
    g = _golden()
    for tag in ("d25", "d300"):
        k2i = dict(zip(g[tag + "_keys"].tolist(), g[tag + "_rows"].tolist()))
        strings = g[tag + "_strings"].tolist()
        for dt in ("f32", "f64"):
            V = g[f"{tag}_vectors_{dt}"]
            got = go.embed(k2i, V, strings)
            assert np.array_equal(go.bits(got), go.bits(_ref_embed(RefGensim, sorted(k2i, key=k2i.get), V, strings, k2i)))


def test_restatement_equals_golden_embed():
    g = _golden()
    for tag in ("d25", "d300"):
        k2i = dict(zip(g[tag + "_keys"].tolist(), g[tag + "_rows"].tolist()))
        strings = g[tag + "_strings"].tolist()
        assert any(not s.isascii() for s in strings)
        for dt in ("f32", "f64"):
            got = go.embed(k2i, g[f"{tag}_vectors_{dt}"], strings)
            assert np.array_equal(go.bits(got), go.bits(g[f"{tag}_embed_{dt}"])), (tag, dt)
    assert np.array_equal(g["d25_vectors_f64"], g["d25_vectors_f32"].astype(np.float64))


# ---- the matcher's host logic ----------------------------------------------------------------------------------------------------
def _kv(d=4, dtype=np.float32, n=3):
    return go.KeyedVectorsStandIn([f"w{i}" for i in range(n)], np.ones((n, d), dtype))


def test_string_model_without_gensim_raises_module_not_found():
    from polyfuzz_b200 import GensimEmbeddings
    try:
        import gensim.downloader  # noqa: F401
        pytest.skip("gensim is installed")
    except ModuleNotFoundError:
        pass
    with pytest.raises(ModuleNotFoundError):
        GensimEmbeddings("glove-twitter-25")


def test_constructor_refusals():
    from polyfuzz_b200 import GensimEmbeddings
    for bad in (42, None, {"a": 1}, np.ones((3, 4))):
        with pytest.raises(ValueError, match="correct Gensim model"):
            GensimEmbeddings(bad)

    class FastTextKeyedVectors(go.KeyedVectorsStandIn):
        pass
    with pytest.raises(NotImplementedError, match="FastText"):
        GensimEmbeddings(FastTextKeyedVectors(["a"], np.ones((1, 4), np.float32)))
    ft = _kv(); ft.buckets_word = {}
    with pytest.raises(NotImplementedError, match="FastText"):
        GensimEmbeddings(ft)
    with pytest.raises(ValueError, match="dimension 1"):
        GensimEmbeddings(_kv(d=1))
    with pytest.raises(ValueError, match="float16"):
        GensimEmbeddings(_kv(dtype=np.float16))
    with pytest.raises(ValueError, match="empty"):
        GensimEmbeddings(_kv(n=0))
    with pytest.raises(ValueError, match="precision"):
        GensimEmbeddings(_kv(), precision="fp32")
    m = GensimEmbeddings(_kv(dtype=np.float64), min_similarity=0.5, top_n=3, cosine_method="knn", model_id="g", precision="fp64")
    assert (m.type, m.model_id, m.min_similarity, m.top_n, m.cosine_method, m.precision) == ("Embeddings", "g", 0.5, 3, "knn", "fp64")
    assert m._wv is None and m.embeddings_to is None and not m.distributed


def test_table_capacity_is_checked_before_any_device_work():
    from polyfuzz_b200 import wordvec
    k2i = {"a": 0, "b": 1, "c": 2}
    V = np.ones((3, 2), np.float32)
    for cap in (3, 6, 2):
        with pytest.raises(ValueError, match="power of two"):
            wordvec.WordVectors(k2i, V, cap=cap)
    with pytest.raises(ValueError, match="outside"):
        wordvec.WordVectors({"a": 3}, V)
    assert [wordvec.default_cap(n) for n in (1, 2, 3, 4, 5, 1000)] == [2, 4, 8, 8, 16, 2048]


def test_pickle_drops_the_device_vocabulary_and_keeps_embeddings_to():
    from polyfuzz_b200 import GensimEmbeddings
    m = GensimEmbeddings(_kv(), top_n=2)
    m._wv = object()                                        # stands for the device vocabulary
    m.embeddings_to = torch.arange(8, dtype=torch.float64).reshape(4, 2)
    st = pickle.loads(pickle.dumps(m))
    assert st._wv is None and m._wv is not None
    assert isinstance(st.embeddings_to, np.ndarray) and st.embeddings_to.dtype == np.float64
    assert np.array_equal(st.embeddings_to, m.embeddings_to.numpy())
    assert st.embedding_model.key_to_index == m.embedding_model.key_to_index and st.top_n == 2
