"""GensimEmbeddings on the GPU: the pooled matrix of K6 (csrc/pfz_wordvec.cu) equals the numpy restatement of the reference's
_embed (tests/gensim_oracle.py) bit for bit, and the matcher's frames equal Embeddings.match on the restated matrices and the
reference's own frames (tests/golden/gensim_c1.npz)."""
import json
import os
import pickle
import threading

import numpy as np
import pandas as pd
import pytest
import torch

import gensim_oracle as go

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "gensim_c1.npz")
REF = os.path.join(ROOT, "oracle", "_ref")
FROM = ["apple", "apples", "appl", "recal", "house", "similarity"]            # the README lists
TO = ["apple", "apples", "mouse"]


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLDEN)
    return {k: z[k] for k in z.files}


def _vocab(g, tag, dt="f32"):
    k2i = dict(zip(g[tag + "_keys"].tolist(), g[tag + "_rows"].tolist()))
    return go.KeyedVectorsStandIn(sorted(k2i, key=k2i.get), g[f"{tag}_vectors_{dt}"], k2i)


def _pool(k2i, V, strings, cap=None):
    from polyfuzz_b200 import wordvec
    out = wordvec.WordVectors(k2i, V, cap=cap).pool(strings)
    assert out.dtype == torch.float64 and out.is_cuda and tuple(out.shape) == (len(strings), V.shape[1])
    return out.cpu().numpy()


def _assert_bits(got, want):
    bad = np.nonzero((go.bits(got) != go.bits(want)).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} rows differ, first {bad[:5].tolist()}"


# ---- K6 against the restatement -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [2, 25, 31, 32, 33, 300])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("with_empty", [False, True])
def test_pool_equals_restatement_on_edge_cases(d, dtype, with_empty):
    keys = [k for k in go.EDGE_KEYS if (with_empty or k != "") and k != "mouse"]
    V = go.random_vectors(len(keys) + 3, d, seed=d, dtype=dtype)       # three rows no key maps to
    rows = np.random.default_rng(d).permutation(len(keys) + 3)[:len(keys)]
    k2i = {k: int(r) for k, r in zip(keys, rows)}
    strings = go.edge_strings()
    _assert_bits(_pool(k2i, V, strings), go.embed(k2i, V, strings))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_pool_at_the_tightest_table(dtype):
    """Keys with "", prefixes of each other and last-code-point neighbours, padded with filler keys to cap - 1 so that the
    table has a single empty slot and probe chains run long."""
    keys, strings = go.prefix_vocab()
    cap = 1 << int(len(keys)).bit_length()
    keys = keys + [f"filler{i}" for i in range(cap - 1 - len(keys))]
    assert len(keys) == cap - 1
    V = go.random_vectors(len(keys), 33, seed=11, dtype=dtype)
    k2i = {k: i for i, k in enumerate(keys)}
    strings = strings + ["filler1 filler12 filler", " ".join(keys[::7])]
    want = go.embed(k2i, V, strings)
    _assert_bits(_pool(k2i, V, strings, cap=cap), want)
    _assert_bits(_pool(k2i, V, strings), want)


def test_pool_equals_golden_reference_embed(golden):
    for tag in ("d25", "d300"):
        strings = golden[tag + "_strings"].tolist()
        for dt in ("f32", "f64"):
            kv = _vocab(golden, tag, dt)
            _assert_bits(_pool(kv.key_to_index, kv.vectors, strings), golden[f"{tag}_embed_{dt}"])


def test_pool_of_an_empty_list_and_lookup_rows():
    from polyfuzz_b200 import wordvec
    wv = wordvec.WordVectors({"a": 1, "b": 0}, np.ones((2, 4), np.float32))
    assert tuple(wv.pool([]).shape) == (0, 4)
    tok_off, tok_row = wv.lookup(["a b", "", " c a"])
    assert tok_off.cpu().tolist() == [0, 2, 3, 6]
    assert tok_row[:6].cpu().tolist() == [1, 0, -1, -1, -1, 1]


# ---- the matcher ----------------------------------------------------------------------------------------------------------------
def _frame_equal(a, b):
    pd.testing.assert_frame_equal(a.reset_index(drop=True), b.reset_index(drop=True), check_exact=True)


@pytest.fixture(scope="module")
def titles(golden):
    strings = golden["d25_strings"].tolist()[9:]
    return strings[:120], strings[120:]


@pytest.mark.parametrize("precision", ["bf16", "fp64"])
@pytest.mark.parametrize("top_n", [1, 10, 40])
@pytest.mark.parametrize("method", ["sparse", "sklearn", "knn"])
def test_match_equals_embeddings_on_the_restated_matrices(golden, titles, precision, top_n, method):
    from polyfuzz_b200 import Embeddings, GensimEmbeddings
    kv = _vocab(golden, "d25")
    frm, to = titles
    ef, et = go.embed(kv.key_to_index, kv.vectors, frm), go.embed(kv.key_to_index, kv.vectors, to)
    for ms in (0.0, 0.75):
        kw = dict(min_similarity=ms, top_n=top_n, cosine_method=method, precision=precision)
        m = GensimEmbeddings(kv, **kw)
        _frame_equal(m.match(frm, to), Embeddings(**kw).match(frm, to, embeddings_from=ef, embeddings_to=et))
        _frame_equal(m.match(frm), Embeddings(**kw).match(frm, None, embeddings_from=ef, embeddings_to=ef))


def test_fp64_frames_equal_the_reference_frames(golden, titles):
    from polyfuzz_b200 import GensimEmbeddings
    lists = {"readme": (FROM, TO), "titles": titles}
    n = 0
    for key in golden:
        if not key.endswith("_frame"):
            continue
        tag, lname, mode, top, ms = key[:-len("_frame")].split("_")
        frm, to = lists[lname]
        m = GensimEmbeddings(_vocab(golden, tag), min_similarity=float(ms[2:]), top_n=int(top[3:]), cosine_method="sklearn",
                             precision="fp64")
        df = m.match(frm, to) if mode == "two" else m.match(frm)
        ref = json.loads(str(golden[key]))
        assert list(df.columns) == list(ref), key
        for c in ref:
            if c.startswith("Similarity"):
                assert np.array_equal(df[c].to_numpy(dtype=np.float64), np.array(ref[c], dtype=np.float64)), (key, c)
            else:                                           # the fixture stores blank cells as None (df_to_json)
                assert [None if isinstance(v, float) and np.isnan(v) else v for v in df[c].tolist()] == ref[c], (key, c)
        n += 1
    assert n == 3 * 12


def test_self_match_pools_once_and_pickle_keeps_re_train_false(golden, titles, monkeypatch):
    from polyfuzz_b200 import GensimEmbeddings, wordvec
    frm, to = titles
    m = GensimEmbeddings(_vocab(golden, "d25"), min_similarity=0.0, top_n=3, precision="fp64")
    calls = []
    pool = wordvec.WordVectors.pool
    monkeypatch.setattr(wordvec.WordVectors, "pool", lambda self, s: calls.append(len(s)) or pool(self, s))
    m.match(to)
    assert calls == [len(to)]
    m.match(frm, to)
    want = m.match(frm[:50], to, re_train=False)
    loaded = pickle.loads(pickle.dumps(m))
    assert loaded._wv is None and isinstance(loaded.embeddings_to, np.ndarray)
    _frame_equal(loaded.match(frm[:50], to, re_train=False), want)


def test_polyfuzz_fit_transform_through_the_reference_orchestrator(golden, titles):
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference orchestrator) was not built")
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    go.install_gensim(REF)
    from polyfuzz import PolyFuzz
    from polyfuzz_b200 import GensimEmbeddings
    frm, to = titles
    kv = _vocab(golden, "d25")
    model = PolyFuzz(GensimEmbeddings(kv, min_similarity=0.0, top_n=2)).fit(to)
    got = model.transform(frm)
    assert list(got) == ["Embeddings"]
    _frame_equal(got["Embeddings"], GensimEmbeddings(kv, min_similarity=0.0, top_n=2).match(frm, to))


@pytest.mark.parametrize("G", [2, 3])
@pytest.mark.parametrize("precision", ["bf16", "fp64"])
def test_distributed_ranks_return_the_single_gpu_frame(golden, titles, G, precision, monkeypatch):
    from test_gpu_tfidf_dist_vocab import run_ok
    from polyfuzz_b200 import GensimEmbeddings
    from polyfuzz_b200.matchers import _embeddings
    frm, to = titles
    kv = _vocab(golden, "d25")
    local = threading.local()
    monkeypatch.setattr(_embeddings, "get_comm", lambda: local.comm)
    for two in (True, False):
        want = GensimEmbeddings(kv, min_similarity=0.0, top_n=10, precision=precision).match(frm, to if two else None)

        def rank(comm):
            local.comm = comm
            return GensimEmbeddings(kv, min_similarity=0.0, top_n=10, precision=precision, distributed=True).match(frm, to if two else None)
        for df in run_ok(G, rank):
            _frame_equal(df, want)
