"""GensimEmbeddings with a FastText model on the GPU: the pooled matrix of K6's pfz_ft_pool (csrc/pfz_wordvec.cu) equals the
restatement of gensim 4's get_vector and the reference's _embed (tests/fasttext_oracle.py) bit for bit, and the matcher's
frames equal Embeddings.match on the restated matrices and the reference's own frames (tests/golden/fasttext_c1.npz)."""
import functools
import json
import os
import pickle
import threading

import numpy as np
import pandas as pd
import pytest
import torch

import fasttext_oracle as fo
import gensim_oracle as go

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "fasttext_c1.npz")
REF = os.path.join(ROOT, "oracle", "_ref")
FROM = ["apple", "apples", "appl", "recal", "house", "similarity"]            # the README lists
TO = ["apple", "apples", "mouse"]
MIN_MAX = [(3, 6), (1, 1), (1, 3), (2, 2), (0, 2), (4, 3), (5, 40)]


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLDEN)
    return {k: z[k] for k in z.files}


@functools.lru_cache(maxsize=4)
def _ngram_table(bucket, d):
    return go.random_vectors(bucket, d, seed=bucket + d)


def _model(d, min_n, max_n, bucket):
    keys, strings = fo.edge_vocab()
    rows = np.random.default_rng(d + bucket).permutation(len(keys) + 3)[:len(keys)]       # three rows no key maps to
    V = go.random_vectors(len(keys) + 3, d, seed=d)
    k2i = {k: int(r) for k, r in zip(keys, rows)}
    NG = _ngram_table(max(bucket, 1), d)[:bucket]
    return fo.FastTextKeyedVectors(sorted(k2i, key=k2i.get), V, NG, min_n, max_n, bucket, k2i), strings


def _pool(ft, strings):
    from polyfuzz_b200 import wordvec
    wv = wordvec.WordVectors(ft.key_to_index, ft.vectors, vectors_ngrams=ft.vectors_ngrams, min_n=ft.min_n, max_n=ft.max_n,
                             bucket=ft.bucket)
    out = wv.pool(strings)
    assert out.dtype == torch.float64 and out.is_cuda and tuple(out.shape) == (len(strings), ft.vectors.shape[1])
    return out.cpu().numpy()


def _assert_bits(got, want):
    bad = np.nonzero((go.bits(got) != go.bits(want)).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} rows differ, first {bad[:5].tolist()}"


# ---- pfz_ft_pool against the restatement --------------------------------------------------------------------------------------
@pytest.mark.parametrize("min_n,max_n", MIN_MAX)
@pytest.mark.parametrize("bucket", [1, 7, 2_000_003])
def test_pool_equals_restatement(min_n, max_n, bucket):
    ft, strings = _model(33, min_n, max_n, bucket)
    _assert_bits(_pool(ft, strings), fo.embed(ft, strings))


@pytest.mark.parametrize("d", [2, 31, 32, 33, 300])
@pytest.mark.parametrize("bucket", [7, 2003])
def test_pool_equals_restatement_across_widths(d, bucket):
    ft, strings = _model(d, 3, 6, bucket)
    _assert_bits(_pool(ft, strings), fo.embed(ft, strings))


def test_pool_equals_the_reference_embed():
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference) was not built")
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    if not go.install_gensim(REF):
        pytest.skip("a real gensim is installed: the reference needs its own KeyedVectors there")
    from polyfuzz.models._gensim import GensimEmbeddings as RefGensim
    for mn, mx in ((3, 6), (1, 3)):
        ft, strings = _model(31, mn, mx, 7)
        strings = [s for s in strings if len(s) < 3000]
        _assert_bits(_pool(ft, strings), np.asarray(RefGensim(ft)._embed(strings), np.float64))


def test_bucket_zero_pools_as_keyed_vectors():
    ft, strings = _model(33, 3, 6, 0)
    got = _pool(ft, strings)
    _assert_bits(got, go.embed(ft.key_to_index, ft.vectors, strings))
    # a row with an unknown token pools in float64: not every entry is a float32 value
    assert (got.astype(np.float32).astype(np.float64) != got).any()


def test_pool_equals_golden_reference_embed(golden):
    ft = fo.golden_model(golden)
    _assert_bits(_pool(ft, golden["strings"].tolist()), golden["embed"])


def test_surrogate_raises_unicode_encode_error():
    from polyfuzz_b200 import GensimEmbeddings
    ft, _ = _model(4, 3, 6, 7)
    with pytest.raises(UnicodeEncodeError):
        GensimEmbeddings(ft, min_similarity=0.0).match(["apple", "x\ud800"], ["apple"])


# ---- the matcher ----------------------------------------------------------------------------------------------------------------
def _frame_equal(a, b):
    pd.testing.assert_frame_equal(a.reset_index(drop=True), b.reset_index(drop=True), check_exact=True)


@pytest.fixture(scope="module")
def titles(golden):
    strings = golden["strings"].tolist()[9:]
    return strings[:120], strings[120:]


@pytest.mark.parametrize("precision", ["bf16", "fp64"])
@pytest.mark.parametrize("top_n", [1, 10, 40])
def test_match_equals_embeddings_on_the_restated_matrices(golden, titles, precision, top_n):
    from polyfuzz_b200 import Embeddings, GensimEmbeddings
    ft = fo.golden_model(golden)
    frm, to = titles
    ef, et = fo.embed(ft, frm), fo.embed(ft, to)
    for ms in (0.0, 0.75):
        kw = dict(min_similarity=ms, top_n=top_n, precision=precision)
        m = GensimEmbeddings(ft, **kw)
        _frame_equal(m.match(frm, to), Embeddings(**kw).match(frm, to, embeddings_from=ef, embeddings_to=et))
        _frame_equal(m.match(frm), Embeddings(**kw).match(frm, None, embeddings_from=ef, embeddings_to=ef))


def test_fp64_frames_equal_the_reference_frames(golden, titles):
    from polyfuzz_b200 import GensimEmbeddings
    lists = {"readme": (FROM, TO), "titles": titles}
    ft = fo.golden_model(golden)
    n = 0
    for key in golden:
        if not key.endswith("_frame"):
            continue
        lname, mode, top, ms = key[:-len("_frame")].split("_")
        frm, to = lists[lname]
        m = GensimEmbeddings(ft, min_similarity=float(ms[2:]), top_n=int(top[3:]), cosine_method="sklearn", precision="fp64")
        df = m.match(frm, to) if mode == "two" else m.match(frm)
        ref = json.loads(str(golden[key]))
        assert list(df.columns) == list(ref), key
        for c in ref:
            if c.startswith("Similarity"):
                assert np.array_equal(df[c].to_numpy(dtype=np.float64), np.array(ref[c], dtype=np.float64)), (key, c)
            else:                                           # the fixture stores blank cells as None (df_to_json)
                assert [None if isinstance(v, float) and np.isnan(v) else v for v in df[c].tolist()] == ref[c], (key, c)
        n += 1
    assert n == 2 * 12


def test_pickle_keeps_re_train_false(golden, titles):
    from polyfuzz_b200 import GensimEmbeddings
    frm, to = titles
    m = GensimEmbeddings(fo.golden_model(golden), min_similarity=0.0, top_n=3, precision="fp64")
    m.match(frm, to)
    want = m.match(frm[:50], to, re_train=False)
    loaded = pickle.loads(pickle.dumps(m))
    assert loaded._wv is None and isinstance(loaded.embeddings_to, np.ndarray)
    _frame_equal(loaded.match(frm[:50], to, re_train=False), want)
    _frame_equal(loaded.match(frm[:50], to), want)                  # re-pooled from the restaged tables


def test_polyfuzz_fit_transform_through_the_reference_orchestrator(golden, titles):
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference orchestrator) was not built")
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    go.install_gensim(REF)
    from polyfuzz import PolyFuzz
    from polyfuzz_b200 import GensimEmbeddings
    frm, to = titles
    ft = fo.golden_model(golden)
    model = PolyFuzz(GensimEmbeddings(ft, min_similarity=0.0, top_n=2)).fit(to)
    got = model.transform(frm)
    assert list(got) == ["Embeddings"]
    _frame_equal(got["Embeddings"], GensimEmbeddings(ft, min_similarity=0.0, top_n=2).match(frm, to))


@pytest.mark.parametrize("G", [2, 3])
@pytest.mark.parametrize("precision", ["bf16", "fp64"])
def test_distributed_ranks_return_the_single_gpu_frame(golden, titles, G, precision, monkeypatch):
    from test_gpu_tfidf_dist_vocab import run_ok
    from polyfuzz_b200 import GensimEmbeddings
    from polyfuzz_b200.matchers import _embeddings
    frm, to = titles
    ft = fo.golden_model(golden)
    local = threading.local()
    monkeypatch.setattr(_embeddings, "get_comm", lambda: local.comm)
    for two in (True, False):
        want = GensimEmbeddings(ft, min_similarity=0.0, top_n=10, precision=precision).match(frm, to if two else None)

        def rank(comm):
            local.comm = comm
            return GensimEmbeddings(ft, min_similarity=0.0, top_n=10, precision=precision, distributed=True).match(frm, to if two else None)
        for df in run_ok(G, rank):
            _frame_equal(df, want)
