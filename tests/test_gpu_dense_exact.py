"""GPU tests of the Embeddings exact mode (precision="fp64"): indices and scores equal the canonical fp64 oracle
(tests/dense_exact_oracle.py) with ==, and the fp16 filter pass stays inside the accumulation-error term gamma that its
certificate assumes (DESIGN.md 4.6)."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dense_exact_oracle as O                                      # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
REF = os.path.join(ROOT, "oracle", "_ref")
FROM = ["apple", "apples", "appl", "recal", "house", "similarity"]
TO = ["apple", "apples", "mouse"]


def _check_gamma(xs, ys, k, thr, self_match, n_splits):
    """Every filter candidate's fp32 score is within gamma * ||x^|| * ||y^|| of the fp64 dot of the fp16 rows."""
    from polyfuzz_b200 import dense
    ci, cv = dense.candidates_f16(xs, ys, dense.k_cand_for(k), thr, self_match, n_splits=n_splits)
    hx, hy = xs.f16.double(), ys.f16.double()
    ok = ci >= 0
    rows = torch.arange(ci.shape[0], device=ci.device)[:, None].expand_as(ci)[ok]
    cols = ci[ok].long()
    exact = (hx[rows] * hy[cols]).sum(-1)
    bound = xs.d_pad * 2.0 ** -22 * hx[rows].norm(dim=1) * hy[cols].norm(dim=1)
    err = (cv[ok] - exact).abs()
    assert bool((err <= bound).all()), float((err / bound).max())


def _run(xf, yf, k, thr=0.0, self_match=False, n_splits=None, gamma=True):
    from polyfuzz_b200 import dense
    xs = dense.stage_exact(xf)
    ys = xs if self_match else dense.stage_exact(yf)
    idx, val, fb = dense.dense_topk_exact(xs, ys, k, thr, self_match=self_match, n_splits=n_splits)
    oi, ov = O.exact_topk(xf, xf if self_match else yf, k, thr, self_match=self_match)
    gi, gv = idx.cpu().numpy(), val.cpu().numpy()
    bad = np.nonzero((gi != oi).any(1) | (gv != ov).any(1))[0]
    assert len(bad) == 0, (bad[:5], gi[bad[:2]], oi[bad[:2]], gv[bad[:2]], ov[bad[:2]])
    if gamma:
        _check_gamma(xs, ys, k, thr, self_match, n_splits)
    return int(fb.item()), ov


@pytest.mark.parametrize("two_cta", ["0", "1"])
@pytest.mark.parametrize("n_from,n_to,d,k", [(6, 3, 300, 3), (300, 700, 768, 10), (129, 257, 64, 1), (1000, 2500, 96, 32),
                                             (257, 5000, 200, 5), (50, 90, 45, 7), (40, 20, 13, 32)])
def test_exact_topk_equals_oracle(n_from, n_to, d, k, two_cta, monkeypatch):
    monkeypatch.setenv("PFZ_K4_2CTA", two_cta)
    g = torch.Generator().manual_seed(n_from * 7 + d)
    xf = torch.randn(n_from, d, generator=g).numpy(); yf = torch.randn(n_to, d, generator=g).numpy().astype(np.float64)
    nd = min(5, n_to, n_from); yf[:nd] = xf[:nd] * 3.0
    for splits in (None, 1):
        _run(xf, yf, k, 0.0, n_splits=splits)
    _run(xf.astype(np.float64), yf, k, 0.05)


def test_staged_rows_are_the_canonical_normalisation():
    from polyfuzz_b200 import dense
    rng = np.random.default_rng(1)
    x = rng.standard_normal((300, 77)); x[4] = 0.0
    s = dense.stage_exact(x)
    got = s.f64.cpu().numpy()
    assert np.array_equal(got[:, :77], O.canon_normalize(x)) and (got[:, 77:] == 0).all()
    assert np.array_equal(s.f16.cpu().numpy()[:, :77], O.canon_normalize(x).astype(np.float16))
    h = s.f16.double().cpu().numpy()
    assert (s.norm16.cpu().numpy() >= np.linalg.norm(h, axis=1)).all()
    assert (s.err16.cpu().numpy() >= np.linalg.norm(got - h, axis=1)).all()
    assert s.maxima.cpu().numpy().tolist() == [s.norm16.max().item(), s.err16.max().item()]


def test_self_match_threshold_on_a_score_and_zero_rows():
    rng = np.random.default_rng(2)
    x = rng.standard_normal((500, 128)).astype(np.float32)
    x[7] = 0.0; x[11] = x[3]
    _, ov = _run(x, None, 4, 0.0, self_match=True)
    thr = float(ov[0, 1])                                        # exactly an existing canonical score: strictly above it only
    _run(x, None, 4, thr, self_match=True)
    y = rng.standard_normal((900, 128)); y[5] = 0.0
    _run(x, y, 6, thr)


def test_many_copies_force_the_fallback():
    """A to-list with 45 copies of one row: no finite candidate list holds all ties, so rows must take the fallback."""
    rng = np.random.default_rng(3)
    v = rng.standard_normal(96)
    y = rng.standard_normal((3000, 96)); y[100:145] = v
    x = v + 0.05 * rng.standard_normal((64, 96))
    fb, _ = _run(x, y, 5, 0.0)
    assert fb > 0
    # more listed rows than the split workspace holds: the rows beyond it are scored whole by one CTA each
    y2 = rng.standard_normal((300, 32)); y2[10:70] = y2[0]
    x2 = y2[0] + 0.01 * rng.standard_normal((2200, 32))
    fb2, _ = _run(x2, y2, 3, 0.0, gamma=False)
    assert fb2 > 2048


def test_clustered_set():
    rng = np.random.default_rng(4)
    centres = rng.standard_normal((100, 128))
    x = centres[rng.integers(0, 100, 600)] + 0.3 * rng.standard_normal((600, 128))
    y = centres[rng.integers(0, 100, 8000)] + 0.3 * rng.standard_normal((8000, 128))
    _run(x.astype(np.float32), y.astype(np.float32), 10, 0.0)


def test_matcher_frames_equal_the_reference_fixture(golden_dir):
    from polyfuzz_b200 import Embeddings
    f = np.load(os.path.join(golden_dir, "dense_c1.npz"))
    for top_n in (1, 2, 3):
        ref = json.load(open(os.path.join(golden_dir, f"dense_c1_top{top_n}.json")))
        df = Embeddings(min_similarity=0.0, top_n=top_n, precision="fp64").match(FROM, TO, f["from_vec"], f["to_vec"])
        assert list(df.columns) == list(ref.keys())
        for c in df.columns:
            assert [None if (isinstance(v, float) and np.isnan(v)) else v for v in df[c].tolist()] == ref[c], c


def _embed(strings):
    """Deterministic stand-in embedder: one seeded Gaussian vector per distinct string."""
    out = []
    for s in strings:
        seed = int.from_bytes(hashlib.sha256(s.encode()).digest()[:8], "little")
        out.append(np.random.default_rng(seed).standard_normal(64))
    return np.array(out)


def test_through_the_reference_orchestrator():
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference orchestrator) was not built")
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    from oracle import ref_shim
    ref_shim.REFERENCE_ROOT = REF
    ref_shim.install()
    from polyfuzz import PolyFuzz
    from polyfuzz_b200 import Embeddings
    from oracle.assemble import assemble
    m = Embeddings(embedding_method=_embed, min_similarity=0.0, precision="fp64", model_id="B200")
    matches = PolyFuzz(m).match(FROM, TO).get_matches()
    oi, ov = O.exact_topk(_embed(FROM), _embed(TO), 1, 0.0)
    exp = assemble(FROM, TO, oi, ov)
    assert matches["To"].tolist() == exp["To"].tolist() and matches["Similarity"].tolist() == exp["Similarity"].tolist()
    model = PolyFuzz(Embeddings(embedding_method=_embed, min_similarity=0.0, precision="fp64")).fit(FROM, TO)
    res = model.transform(TO)
    df = res[list(res.keys())[0]]
    oi, ov = O.exact_topk(_embed(TO), _embed(TO), 1, 0.0)
    assert df["To"].tolist() == [TO[j] if v >= 0.001 else None for j, v in zip(oi[:, 0], ov[:, 0])]


def test_c4_shape_sampled_rows():
    """100k x 100k x 768, the C4 inputs (torch seeds 0 / 1), top-10: 200 sampled rows equal the oracle."""
    from polyfuzz_b200 import dense
    n, d, k = 100_000, 768, 10
    dev = torch.device("cuda")
    torch.manual_seed(0); X = torch.randn(n, d, device=dev)
    torch.manual_seed(1); Y = torch.randn(n, d, device=dev)
    xs, ys = dense.stage_exact(X), dense.stage_exact(Y)
    idx, val, fb = dense.dense_topk_exact(xs, ys, k, 0.0)
    rows = np.random.default_rng(0).choice(n, 200, replace=False)
    xn = xs.f64[torch.from_numpy(rows).to(dev)].cpu().numpy(); yn = ys.f64.cpu().numpy()
    assert np.array_equal(yn[:1000], O.canon_normalize(Y[:1000].double().cpu().numpy()))
    assert np.array_equal(xn, O.canon_normalize(X[torch.from_numpy(rows).to(dev)].double().cpu().numpy()))
    oi, ov = O.exact_topk(xn, yn, k, 0.0, normalized=True, block=4)
    assert np.array_equal(idx.cpu().numpy()[rows], oi) and np.array_equal(val.cpu().numpy()[rows], ov)
    print(f"C4 exact: fallback rows {int(fb.item())}")
