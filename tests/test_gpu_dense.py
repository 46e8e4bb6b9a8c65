"""GPU tests of K4 (dense bf16 wgmma cosine top-k) against an fp64 reference computed from the SAME
bf16-rounded inputs.  Tolerance (north_star): scores within 1e-5; indices must be an exact top-k of the fp64
scores up to that tolerance (every returned score >= k-th fp64 score - 2e-5, ordered descending)."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _check(x_bf16, y_bf16, idx, val, k, min_sim=0.0, self_match=False):
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
        # near the threshold the fp32 accumulation may differ from fp64 by < TOL
        assert abs(int(valid.sum()) - cnt_ref) <= int(((np.abs(s[i] - min_sim) < 2 * TOL)).sum()), (i, valid.sum(), cnt_ref)
        g = got[valid]
        assert len(set(g.tolist())) == len(g)
        np.testing.assert_allclose(val[i][valid], s[i][g], atol=TOL, rtol=0)
        assert (np.diff(val[i][valid]) <= 0).all()
        if len(g) and cnt_ref:
            assert s[i][g].min() >= ref_sorted[i][min(len(g), cnt_ref) - 1] - 2 * TOL


@pytest.mark.parametrize("two_cta", ["0", "1"])
@pytest.mark.parametrize("n_from,n_to,d,k", [(6, 3, 300, 3), (300, 700, 768, 10), (129, 257, 64, 1), (1000, 2500, 96, 32), (257, 5000, 200, 5)])
def test_dense_topk_random(n_from, n_to, d, k, two_cta, monkeypatch):
    """Both launch shapes: one CTA per 128 from-rows, and CTA pairs (cluster of 2 sharing each to-tile through TMA multicast)."""
    from polyfuzz_b200 import dense
    monkeypatch.setenv("PFZ_K4_2CTA", two_cta)
    g = torch.Generator().manual_seed(n_from * 7 + d)
    xf = torch.randn(n_from, d, generator=g); yf = torch.randn(n_to, d, generator=g)
    nd = min(5, n_to, n_from); yf[:nd] = xf[:nd] * 3.0           # exact duplicates (up to scale) -> score 1.0
    x, _ = dense.to_bf16_rows(xf.numpy(), True); y, _ = dense.to_bf16_rows(yf.numpy().astype(np.float64), True)
    kk = min(k, n_to)
    for splits in (None, 1):
        idx, val = dense.dense_topk(x, y, kk, 0.0, n_splits=splits)
        _check(x, y, idx, val, kk)
    idx, val = dense.dense_topk(x, y, kk, 0.05)
    _check(x, y, idx, val, kk, min_sim=0.05)


def test_dense_self_match_and_fixture(golden_dir):
    from polyfuzz_b200 import dense, Embeddings
    g = torch.Generator().manual_seed(5)
    xf = torch.randn(500, 128, generator=g)
    x, _ = dense.to_bf16_rows(xf.numpy(), True)
    idx, val = dense.dense_topk(x, x, 4, 0.0, self_match=True)
    assert (idx.cpu().numpy() != np.arange(500)[:, None]).all()
    _check(x, x, idx, val, 4, self_match=True)
    # the reference's own dense fixture (tests/from_list.npy, tests/to_list.npy) and its sklearn-branch result
    f = np.load(os.path.join(golden_dir, "dense_c1.npz"))
    frm = ["apple", "apples", "appl", "recal", "house", "similarity"]; to = ["apple", "apples", "mouse"]
    for top_n in (1, 2, 3):
        ref = json.load(open(os.path.join(golden_dir, f"dense_c1_top{top_n}.json")))
        df = Embeddings(min_similarity=0.0, top_n=top_n).match(frm, to, f["from_vec"], f["to_vec"])
        assert list(df.columns) == list(ref.keys())
        for c in df.columns:
            if c.startswith("Similarity"):
                np.testing.assert_allclose(df[c].to_numpy(), np.array(ref[c], dtype=float), atol=2e-3)   # bf16 inputs, 3-dp rounding
            elif c != "From":
                pass
        assert df["To"].tolist() == ref["To"]
