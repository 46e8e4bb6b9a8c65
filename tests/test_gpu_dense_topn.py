"""GPU tests of Embeddings top_n > 32 (DESIGN.md 4.7: bound pass, threshold pass, select), both precisions.  The exact mode
equals the canonical fp64 oracle (tests/dense_exact_oracle.py) with ==; the bf16 mode equals `dense_topk` bit for bit where
both apply and is otherwise checked against an fp64 product of the same bf16 rows."""
import hashlib
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
TOL = 1e-5


def _check(x_bf16, y_bf16, idx, val, k, min_sim=0.0, self_match=False):
    """Copy of test_gpu_dense._check: an exact top-k of the fp64 scores of the bf16 rows up to the fp32 accumulation."""
    x = x_bf16.double(); y = y_bf16.double()
    s = (x @ y.T).cpu().numpy()
    idx = idx.cpu().numpy(); val = val.cpu().numpy()
    n, m = s.shape
    if self_match:
        s[np.arange(min(n, m)), np.arange(min(n, m))] = -np.inf
    s_ok = np.where(s > min_sim, s, -np.inf)
    ref_sorted = -np.sort(-s_ok, axis=1)[:, :k]
    for i in range(n):
        got = idx[i]; valid = got >= 0
        cnt_ref = int(np.isfinite(ref_sorted[i]).sum())
        assert abs(int(valid.sum()) - cnt_ref) <= int(((np.abs(s[i] - min_sim) < 2 * TOL)).sum()), (i, valid.sum(), cnt_ref)
        g = got[valid]
        assert len(set(g.tolist())) == len(g)
        np.testing.assert_allclose(val[i][valid], s[i][g], atol=TOL, rtol=0)
        assert (np.diff(val[i][valid]) <= 0).all()
        if len(g) and cnt_ref:
            assert s[i][g].min() >= ref_sorted[i][min(len(g), cnt_ref) - 1] - 2 * TOL


def _exact(xf, yf, k, thr=0.0, self_match=False, oracle=None, **kw):
    """GPU exact top-k (k > 32 through dense_topk_exact, else dense_topn_bounded) == the oracle.  Returns (overflow rows, oracle)."""
    from polyfuzz_b200 import dense
    xs = dense.stage_exact(xf)
    ys = xs if self_match else dense.stage_exact(yf)
    if k > 32 and not kw:
        idx, val, n_over = dense.dense_topk_exact(xs, ys, k, thr, self_match=self_match)
        n_over = int(n_over.item())
    else:
        idx, val, n_over = dense.dense_topn_bounded(xs, ys, k, thr, self_match=self_match, **kw)
    if oracle is None:
        oracle = O.exact_topk(xf, xf if self_match else yf, k, thr, self_match=self_match)
    oi, ov = oracle[0][:, :k], oracle[1][:, :k]
    gi, gv = idx.cpu().numpy(), val.cpu().numpy()
    bad = np.nonzero((gi != oi).any(1) | (gv != ov).any(1))[0]
    assert len(bad) == 0, (k, bad[:5], gi[bad[:1]], oi[bad[:1]], gv[bad[:1]], ov[bad[:1]])
    return n_over, oracle


@pytest.mark.parametrize("two_cta", ["0", "1"])
@pytest.mark.parametrize("n_from,n_to,d", [(6, 3, 300), (300, 700, 768), (129, 257, 64), (1000, 2500, 96), (257, 5000, 200), (50, 90, 45),
                                           (40, 20, 13)])
def test_exact_topn_equals_oracle(n_from, n_to, d, two_cta, monkeypatch):
    monkeypatch.setenv("PFZ_K4_2CTA", two_cta)
    g = torch.Generator().manual_seed(n_from * 7 + d)
    xf = torch.randn(n_from, d, generator=g).numpy(); yf = torch.randn(n_to, d, generator=g).numpy().astype(np.float64)
    nd = min(5, n_to, n_from); yf[:nd] = xf[:nd] * 3.0
    o32 = O.exact_topk(xf, yf, 300, 0.0)
    o64 = O.exact_topk(xf.astype(np.float64), yf, 300, 0.05)
    for k in (33, 64, 100, 300):
        _exact(xf, yf, k, 0.0, oracle=o32)
        _exact(xf.astype(np.float64), yf, k, 0.05, oracle=o64)


def test_exact_topn_self_match_threshold_on_a_score_and_zero_rows():
    rng = np.random.default_rng(2)
    x = rng.standard_normal((500, 128)).astype(np.float32)
    x[7] = 0.0; x[11] = x[3]
    _, (oi, ov) = _exact(x, None, 40, 0.0, self_match=True)
    thr = float(ov[0, 20])                                        # exactly an existing canonical score: strictly above it only
    _exact(x, None, 40, thr, self_match=True)
    y = rng.standard_normal((900, 128)); y[5] = 0.0
    _exact(x, y, 64, thr)


def _clustered(rng, n_x, n_y, d, n_c=50, noise=0.3):
    centres = rng.standard_normal((n_c, d))
    cx, cy = rng.integers(0, n_c, n_x), rng.integers(0, n_c, n_y)
    x = centres[cx] + noise * rng.standard_normal((n_x, d))
    y = centres[cy] + noise * rng.standard_normal((n_y, d))
    return x, y, cy


def test_exact_topn_clustered_and_sorted_by_centre():
    """Sorted by centre, each row's neighbours sit in one or two to-splits: the bound is loose but must stay right."""
    rng = np.random.default_rng(4)
    x, y, cy = _clustered(rng, 600, 8000, 128)
    for yy in (y, y[np.argsort(cy, kind="stable")]):
        for k in (33, 100):
            _exact(x.astype(np.float32), yy.astype(np.float32), k, 0.0)
        _exact(x, yy, 64, 0.5)


def test_overflow_many_copies_and_small_cap():
    rng = np.random.default_rng(3)
    v = rng.standard_normal(96)
    y = rng.standard_normal((3000, 96)); y[100:500] = v             # 400 copies: more candidates than the default 256 slots
    x = v + 0.05 * rng.standard_normal((64, 96))
    n_over, _ = _exact(x, y, 40, 0.0)
    assert n_over > 0
    x2, y2, _ = _clustered(rng, 300, 4000, 64)
    n_over2, o = _exact(x2, y2, 33, 0.0, cap=40)
    assert n_over2 > 0
    n_over3, _ = _exact(x2, y2, 33, 0.0, oracle=o, cap=40, chunk_rows=100)
    assert n_over3 == n_over2
    # bf16: the copies overflow the default capacity, and the re-run gives the list of a capacity that holds every to-row
    from polyfuzz_b200 import dense
    xb, _ = dense.to_bf16_rows(x, True); yb, _ = dense.to_bf16_rows(y, True)
    i1, v1, n1 = dense.dense_topn_bounded(xb, yb, 40, 0.0)
    i2, v2, n2 = dense.dense_topn_bounded(xb, yb, 40, 0.0, cap=len(y))
    assert n1 > 0 and n2 == 0 and torch.equal(i1, i2) and torch.equal(v1, v2)
    _check(xb, yb, i1, v1, 40)


@pytest.mark.parametrize("two_cta", ["0", "1"])
def test_bf16_bounded_path_equals_dense_topk(two_cta, monkeypatch):
    from polyfuzz_b200 import dense
    monkeypatch.setenv("PFZ_K4_2CTA", two_cta)
    g = torch.Generator().manual_seed(9)
    xf = torch.randn(700, 200, generator=g); yf = torch.randn(5000, 200, generator=g)
    yf[:5] = xf[:5] * 2.0; yf[40:60] = yf[39]                    # exact duplicates and a run of ties
    x, _ = dense.to_bf16_rows(xf.numpy(), True); y, _ = dense.to_bf16_rows(yf.numpy(), True)
    for splits in (None, 1):
        for k in (1, 10, 16, 32):
            ri, rv = dense.dense_topk(x, y, k, 0.0, n_splits=splits)
            gi, gv, _ = dense.dense_topn_bounded(x, y, k, 0.0, n_splits=splits)
            assert torch.equal(gi, ri) and torch.equal(gv, rv), k
        ri, rv = dense.dense_topk(x, y, 32, 0.0, n_splits=splits)
        for k in (33, 100, 300):
            gi, gv = dense.dense_topk(x, y, k, 0.0, n_splits=splits)
            assert torch.equal(gi[:, :32], ri) and torch.equal(gv[:, :32], rv), k
            _check(x, y, gi, gv, k)
    ri, rv = dense.dense_topk(x, x, 16, 0.05, self_match=True)
    gi, gv, _ = dense.dense_topn_bounded(x, x, 16, 0.05, self_match=True)
    assert torch.equal(gi, ri) and torch.equal(gv, rv)
    gi, gv = dense.dense_topk(x, x, 50, 0.05, self_match=True)
    _check(x, x, gi, gv, 50, min_sim=0.05, self_match=True)


def test_degenerate_sizes():
    from polyfuzz_b200 import dense
    rng = np.random.default_rng(5)
    x = rng.standard_normal((70, 48)); y = rng.standard_normal((50, 48))
    _exact(x, y, 64, 0.0)                                        # n_to < k
    _exact(y, None, 49, -1.0, self_match=True)                   # k = n_to - 1 in a self-match: every other row
    _exact(x, y[:3], 40, -1.0)                                   # n_to = 3
    xl = rng.standard_normal((20, 64)); yl = rng.standard_normal((3000, 64))
    _exact(xl, yl, 1024, 0.0)                                    # k = 1024 on a small from-list
    for xx, yy, k, thr, sm in ((x, y, 64, 0.0, False), (y, y, 49, -1.0, True), (x, y[:3], 40, -1.0, False), (xl, yl, 1024, 0.0, False)):
        xb, _ = dense.to_bf16_rows(xx, True)
        yb = xb if sm else dense.to_bf16_rows(yy, True)[0]
        gi, gv = dense.dense_topk(xb, yb, k, thr, self_match=sm)
        _check(xb, yb, gi, gv, k, min_sim=thr, self_match=sm)


def _embed(strings):
    out = []
    for s in strings:
        seed = int.from_bytes(hashlib.sha256(s.encode()).digest()[:8], "little")
        out.append(np.random.default_rng(seed).standard_normal(64))
    return np.array(out)


def test_matcher_frames_top40():
    from polyfuzz_b200 import Embeddings
    from oracle.assemble import assemble
    frm = [f"from {i}" for i in range(90)]
    to = [f"to {i}" for i in range(130)]
    ef, et = _embed(frm), _embed(to)
    cols = ["From"] + [c for r in range(40) for c in (("To", "Similarity") if r == 0 else (f"To_{r + 1}", f"Similarity_{r + 1}"))]
    for precision in ("bf16", "fp64"):
        df = Embeddings(min_similarity=0.0, top_n=40, precision=precision).match(frm, to, ef, et)
        assert list(df.columns) == cols and len(df) == len(frm)
    oi, ov = O.exact_topk(ef, et, 40, 0.0)
    exp = assemble(frm, to, oi, ov)
    df = Embeddings(min_similarity=0.0, top_n=40, precision="fp64").match(frm, to, ef, et)
    for c in cols:
        assert [None if (isinstance(v, float) and np.isnan(v)) else v for v in df[c].tolist()] == list(exp[c]), c
    m = Embeddings(min_similarity=0.0, top_n=40, precision="fp64")
    m.match(frm, to, ef, et)
    df2 = m.match(frm[:10], to, ef[:10], re_train=False)          # transform against the fitted to-embeddings
    for c in cols:
        assert [None if (isinstance(v, float) and np.isnan(v)) else v for v in df2[c].tolist()] == list(exp[c])[:10], c
    dfs = Embeddings(min_similarity=0.0, top_n=40, precision="fp64").match(frm, None, ef)
    si, sv = O.exact_topk(ef, ef, 40, 0.0, self_match=True)
    exps = assemble(frm, None, si, sv)
    assert df.shape == dfs.shape and dfs["To_40"].tolist() == list(exps["To_40"])


def test_through_the_reference_orchestrator_top40():
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference orchestrator) was not built")
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    from oracle import ref_shim
    ref_shim.REFERENCE_ROOT = REF
    ref_shim.install()
    from polyfuzz import PolyFuzz
    from polyfuzz_b200 import Embeddings
    from oracle.assemble import assemble
    frm = [f"item {i}" for i in range(60)]
    to = [f"thing {i}" for i in range(80)]
    m = Embeddings(embedding_method=_embed, min_similarity=0.0, top_n=40, precision="fp64", model_id="B200")
    matches = PolyFuzz(m).match(frm, to).get_matches()
    oi, ov = O.exact_topk(_embed(frm), _embed(to), 40, 0.0)
    exp = assemble(frm, to, oi, ov)
    assert matches["To"].tolist() == exp["To"].tolist() and matches["Similarity"].tolist() == exp["Similarity"].tolist()
    model = PolyFuzz(Embeddings(embedding_method=_embed, min_similarity=0.0, top_n=40, precision="fp64")).fit(frm, to)
    res = model.transform(to)
    df = res[list(res.keys())[0]]
    oi, ov = O.exact_topk(_embed(to), _embed(to), 40, 0.0)
    assert df["To"].tolist() == [to[j] if v >= 0.001 else None for j, v in zip(oi[:, 0], ov[:, 0])]


def test_sharded_to_list_merges_to_the_single_call():
    from polyfuzz_b200 import dense
    from polyfuzz_b200.distributed import merge_topk_any, shard_bounds
    rng = np.random.default_rng(6)
    x = rng.standard_normal((300, 96)); y = rng.standard_normal((2500, 96))
    xs = dense.stage_exact(x)
    ri, rv, _ = dense.dense_topk_exact(xs, dense.stage_exact(y), 64, 0.0)
    parts_i, parts_v = [], []
    for r in range(3):
        lo, hi = shard_bounds(len(y), 3, r)
        i, v, _ = dense.dense_topk_exact(xs, dense.stage_exact(y[lo:hi]), 64, 0.0, to_index_base=lo)
        parts_i.append(i); parts_v.append(v)
    mi, mv = merge_topk_any(torch.stack(parts_i), torch.stack(parts_v), 64)
    assert torch.equal(mi, ri) and torch.equal(mv, rv)


def test_c4_shape_sampled_rows_top100():
    """100k x 100k x 768, the C4 inputs (torch seeds 0 / 1), top-100 in the exact mode: 200 sampled rows equal the oracle."""
    from polyfuzz_b200 import dense
    n, d, k = 100_000, 768, 100
    dev = torch.device("cuda")
    torch.manual_seed(0); X = torch.randn(n, d, device=dev)
    torch.manual_seed(1); Y = torch.randn(n, d, device=dev)
    xs, ys = dense.stage_exact(X), dense.stage_exact(Y)
    idx, val, n_over = dense.dense_topn_bounded(xs, ys, k, 0.0)
    rows = np.random.default_rng(0).choice(n, 200, replace=False)
    xn = xs.f64[torch.from_numpy(rows).to(dev)].cpu().numpy(); yn = ys.f64.cpu().numpy()
    oi, ov = O.exact_topk(xn, yn, k, 0.0, normalized=True, block=4)
    assert np.array_equal(idx.cpu().numpy()[rows], oi) and np.array_equal(val.cpu().numpy()[rows], ov)
    print(f"C4 exact top-100: overflow rows {n_over}")
