"""CPU tests of the Embeddings exact mode: the numpy oracle against a plain-Python statement of the canonical contract,
the oracle against the reference's own dense fixture, and the matcher's `precision` control flow with stubbed kernels."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dense_exact_oracle as O                                      # noqa: E402
from oracle.assemble import assemble                                # noqa: E402

FROM = ["apple", "apples", "appl", "recal", "house", "similarity"]
TO = ["apple", "apples", "mouse"]


def _py_dot(a, b):
    p = [0.0] * 32
    for c in range(len(a)):                                          # c = 32 t + l, ascending t for every lane l
        prod = float(a[c]) * float(b[c])
        p[c % 32] = p[c % 32] + prod
    for o in (16, 8, 4, 2, 1):
        p = [p[l] + p[l ^ o] for l in range(32)]
    return p[0]


def _py_normalize(x):
    ss = _py_dot(x, x)
    if ss == 0.0:
        return [float(v) for v in x]
    n = math.sqrt(ss)
    return [float(v) / n for v in x]


@pytest.mark.parametrize("d", [1, 7, 32, 45, 300])
def test_oracle_dot_and_normalisation_equal_the_definition(d):
    rng = np.random.default_rng(d)
    X = rng.standard_normal((5, d)) * rng.choice([1e-3, 1.0, 1e3], size=(5, 1))
    X[3] = 0.0
    Y = rng.standard_normal((4, d)).astype(np.float32).astype(np.float64)
    got = O.canon_dot(X, Y)
    for i in range(5):
        for j in range(4):
            assert got[i, j] == _py_dot(X[i], Y[j]), (i, j)
    Xn = O.canon_normalize(X)
    for i in range(5):
        assert Xn[i].tolist() == _py_normalize(X[i])
    assert (Xn[3] == 0).all()
    assert O.canon_self_dot(X).tolist() == [_py_dot(x, x) for x in X]


def test_oracle_frames_equal_the_reference_fixture(golden_dir):
    f = np.load(os.path.join(golden_dir, "dense_c1.npz"))
    for top_n in (1, 2, 3):
        ref = json.load(open(os.path.join(golden_dir, f"dense_c1_top{top_n}.json")))
        idx, val = O.exact_topk(f["from_vec"], f["to_vec"], top_n, 0.0)
        df = assemble(FROM, TO, idx, val)
        assert list(df.columns) == list(ref.keys())
        for c in df.columns:
            assert [None if (isinstance(v, float) and np.isnan(v)) else v for v in df[c].tolist()] == ref[c], c


def test_oracle_ranking_threshold_and_self_match():
    X = np.array([[1.0, 0.0], [1.0, 0.0], [0.0, 1.0], [1.0, 1.0]])
    idx, val = O.exact_topk(X, X, 3, 0.0, self_match=True)
    assert idx[0].tolist() == [1, 3, -1] and idx[1].tolist() == [0, 3, -1]       # tie at 1.0 impossible here; 0.0 is not > 0
    assert val[0, 2] == 0.0
    s = val[0, 1]
    idx2, _ = O.exact_topk(X, X, 3, s, self_match=True)                        # strict: a score equal to thr is out
    assert idx2[0].tolist() == [1, -1, -1]


def test_embeddings_precision_dispatch_with_stubbed_kernels(monkeypatch):
    from polyfuzz_b200 import dense, Embeddings
    calls = []

    def fake_stage(x):
        x = np.asarray(x, dtype=np.float64)
        calls.append(("stage", x.shape))
        return O.canon_normalize(x)

    def fake_exact(x, y, k, min_similarity=0.0, self_match=False, from_index_base=0, to_index_base=0, **kw):
        calls.append(("exact", k, self_match))
        idx, val = O.exact_topk(x, y, k, min_similarity, self_match=self_match, normalized=True)
        return torch.from_numpy(idx), torch.from_numpy(val), torch.zeros(1, dtype=torch.int32)

    def no_bf16(*a, **kw):
        raise AssertionError("the bf16 path must not run for precision='fp64'")

    monkeypatch.setattr(dense, "stage_exact", fake_stage)
    monkeypatch.setattr(dense, "dense_topk_exact", fake_exact)
    monkeypatch.setattr(dense, "to_bf16_rows", no_bf16)
    monkeypatch.setattr(dense, "dense_topk", no_bf16)
    with pytest.raises(ValueError):
        Embeddings(precision="fp32")
    assert Embeddings().precision == "bf16"
    rng = np.random.default_rng(0)
    ef, et = rng.normal(size=(4, 8)), rng.normal(size=(3, 8))
    et[1] = ef[2] * 2.0
    frm, to = ["a", "b", "c", "d"], ["x", "y", "z"]
    m = Embeddings(min_similarity=0.0, top_n=2, precision="fp64")
    df = m.match(frm, to, ef, et)
    assert list(df.columns) == ["From", "To", "Similarity", "To_2", "Similarity_2"] and df["To"][2] == "y" and df["Similarity"][2] == 1.0
    assert calls == [("stage", (4, 8)), ("stage", (3, 8)), ("exact", 2, False)]
    calls.clear()
    df2 = m.match(["q"], to, ef[:1], re_train=False)                 # transform: the fitted to-embeddings
    assert calls == [("stage", (1, 8)), ("stage", (3, 8)), ("exact", 2, False)] and len(df2) == 1
    calls.clear()
    df3 = m.match(frm, None, ef)                                      # self-match: one staged matrix for both sides
    assert calls == [("stage", (4, 8)), ("exact", 2, True)] and (df3["To"] != df3["From"]).all()
    calls.clear()
    Embeddings(min_similarity=0.9, top_n=1, precision="fp64", cosine_method="sklearn").match(frm, to, ef, et)
    assert calls[-1] == ("exact", 1, False)
