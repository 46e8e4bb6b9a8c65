"""GPU tests of the exact mode's certificate and bounds at their edges (inputs: tests/dense_cert_cases.py, whose properties
tests/test_oracle_dense_cert.py checks on the CPU).  Every result equals the canonical fp64 oracle (tests/dense_exact_oracle.py)
with ==; the certificate tests also assert which rows take the fallback."""
import math
import os
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dense_cert_cases as C                                          # noqa: E402
import dense_exact_oracle as O                                        # noqa: E402

pytestmark = pytest.mark.gpu
KS = (1, 4, 5, 10, 16, 32)
KS_TOPN = (33, 40, 100)


def _dev(h):
    """dense.ExactRows from a dense_cert_cases.HostRows, unchanged."""
    from polyfuzz_b200 import dense
    s = dense.ExactRows()
    s.f64 = torch.from_numpy(np.ascontiguousarray(h.f64)).cuda()
    s.f16 = torch.from_numpy(np.ascontiguousarray(h.f16)).cuda()
    s.norm16 = torch.from_numpy(np.ascontiguousarray(h.norm16)).cuda()
    s.err16 = torch.from_numpy(np.ascontiguousarray(h.err16)).cuda()
    s.maxima = torch.from_numpy(np.ascontiguousarray(h.maxima)).cuda()
    return s


def _same(gi, gv, oi, ov, what):
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    bad = np.nonzero((gi != oi).any(1) | (gv.view(np.uint64) != ov.view(np.uint64)).any(1))[0]
    assert len(bad) == 0, (what, bad[:5], gi[bad[:1]], oi[bad[:1]], gv[bad[:1]], ov[bad[:1]])


def _exact_all(xh, yh, thr, ks=KS + KS_TOPN, self_match=False, splits=(None, 1)):
    """dense_topk_exact (k <= 32) and dense_topn_bounded (every k) on staged host rows == the oracle on their f64 rows."""
    from polyfuzz_b200 import dense
    xs = _dev(xh)
    ys = xs if self_match else _dev(yh)
    oi, ov = O.exact_topk(xh.f64, xh.f64 if self_match else yh.f64, max(ks), thr, self_match=self_match, normalized=True)
    for sp in splits:
        for k in ks:
            i, v, _ = dense.dense_topk_exact(xs, ys, k, thr, self_match=self_match, n_splits=sp)
            _same(i, v, oi[:, :k], ov[:, :k], ("topk_exact", k, sp, thr))
            i, v, _ = dense.dense_topn_bounded(xs, ys, k, thr, self_match=self_match, n_splits=sp)
            _same(i, v, oi[:, :k], ov[:, :k], ("topn_bounded", k, sp, thr))


def _fallback_rows(xs, ys, k, thr, kc=None):
    """Rows exact_rescore leaves to the fallback, and each row's filter candidate count."""
    from polyfuzz_b200 import dense
    kc = kc or max(k, dense.k_cand_for(k))
    ci, cv = dense.candidates_f16(xs, ys, kc, thr)
    _, _, fb, cnt = dense.exact_rescore(xs, ys, ci, cv, k, thr)
    n = int(cnt.item())
    return sorted(fb[:n].cpu().tolist()), (ci >= 0).sum(1).cpu().numpy(), cv.cpu().numpy()


# ---- staging -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("d", [32, 40, 64])
def test_staging_of_edge_rows(d):
    from polyfuzz_b200 import dense
    rng = np.random.default_rng(d)
    parts = [C.off_norm_rows(d)[0], C.aligned_rows(d, 3, rng), rng.standard_normal((3, d))]
    if d >= 15:
        parts.append(C.fp16_edge_rows(d, rng))
    X = np.vstack(parts)
    with np.errstate(over="ignore"):
        want = C.stage_host(X)
    s = dense.stage_exact(X)
    assert np.array_equal(s.f64.cpu().numpy().view(np.uint64), want.f64.view(np.uint64))      # the sign of zero counts
    assert np.array_equal(s.f16.cpu().numpy().view(np.uint16), want.f16.view(np.uint16))
    h = s.f16.double().cpu().numpy(); f = s.f64.cpu().numpy()
    n16, e16 = s.norm16.cpu().numpy(), s.err16.cpu().numpy()
    for i in range(len(X)):                                 # upper bounds, compared exactly
        assert Fraction(float(n16[i])) ** 2 >= C.sq_norm(h[i]) and Fraction(float(e16[i])) ** 2 >= C.sq_norm(f[i] - h[i])
    assert s.maxima.cpu().numpy().tolist() == [n16.max(), e16.max()]


# ---- gamma -------------------------------------------------------------------------------------------------------------

GAMMA_WORST = {}


def _gamma_ratio(xs, ys, thr=-1.0):
    """max over every filter candidate of |fp32 score - exact x^.y^| / (gamma ||x^|| ||y^||)."""
    from polyfuzz_b200 import dense
    ci, cv = dense.candidates_f16(xs, ys, 32, thr, n_splits=1)
    hx, hy = xs.f16.double(), ys.f16.double()
    ok = ci >= 0
    rows = torch.arange(ci.shape[0], device=ci.device)[:, None].expand_as(ci)[ok]
    cols = ci[ok].long()
    exact = (hx[rows] * hy[cols]).sum(-1)                   # fp64 sum of exact products: its error is ~2^-31 of gamma's
    bound = xs.d_pad * 2.0 ** -22 * hx[rows].norm(dim=1) * hy[cols].norm(dim=1)
    return float(((cv[ok] - exact).abs() / bound).max()), int(ok.sum())


@pytest.mark.parametrize("two_cta", ["0", "1"])
@pytest.mark.parametrize("d", [8, 64, 768, 4096])
def test_gamma_on_same_sign_and_aligned_rows(d, two_cta, monkeypatch):
    monkeypatch.setenv("PFZ_K4_2CTA", two_cta)
    rng = np.random.default_rng(d)
    h = C.same_sign_f16(d, 300, rng)
    hr = C.HostRows(h.astype(np.float64), h)                # only f16 matters to the filter; the bounds stay honest
    r1, n1 = _gamma_ratio(_dev(C.HostRows(hr.f64[:130], h[:130])), _dev(C.HostRows(hr.f64[130:], h[130:])))
    signs = rng.choice([-1.0, 1.0], size=d)
    X = C.aligned_rows(d, 130, rng, signs); Y = C.aligned_rows(d, 170, rng, signs)
    r2, n2 = _gamma_ratio(_dev(C.stage_host(X)), _dev(C.stage_host(Y)))
    assert n1 > 0 and n2 > 0
    GAMMA_WORST[(d, two_cta)] = (r1, r2)
    print(f"gamma d={d} 2cta={two_cta}: worst err / (gamma |x^||y^|) same-sign {r1:.4f}, aligned {r2:.4f}")
    assert r1 <= 1.0 and r2 <= 1.0


# ---- the certificate, k <= 32 ------------------------------------------------------------------------------------------

def test_certificate_fewer_candidates_small_margin_is_certified():
    rng = np.random.default_rng(11)
    Y = rng.standard_normal((300, 64)); X = Y[:6] + 0.05 * rng.standard_normal((6, 64))
    xh, yh = C.stage_host(X), C.stage_host(Y)
    thr = 0.9
    for i in range(6):
        assert xh.margin(i, yh) <= C.exact_margin_max(64)
    fb, nc, _ = _fallback_rows(_dev(xh), _dev(yh), 4, thr)
    print(f"certificate, nc < kc and M_i <= M_max: {len(fb)} fallback rows of 6")
    assert (nc < 10).all() and fb == []
    _exact_all(xh, yh, thr)


@pytest.mark.parametrize("side", ["from", "to"])
def test_certificate_fewer_candidates_large_margin_falls_back(side):
    xh, yh, X, Y, c, thr = C.broken_pair(64, 200, np.random.default_rng(5), side=side)
    xs, ys = _dev(xh), _dev(yh)
    fb, nc, _ = _fallback_rows(xs, ys, 4, thr)
    print(f"certificate, nc < kc and M_i > M_max ({side}): fallback rows {fb} of 4")
    assert nc[0] == 0                                       # the filter dropped the eligible pair (0, 0)
    assert fb == ([0] if side == "from" else [0, 1, 2, 3])  # a pushed to-row raises every from-row's M_i
    _exact_all(xh, yh, thr)
    _exact_all(xh, yh, 0.0)


def test_certificate_b_at_thr_boundary():
    """thr = B (the row's bound, computed from its kc-th filter score) certifies by B <= thr; one double below, k = kc, it
    cannot (the k-th canonical score lies below B) and the row falls back."""
    from polyfuzz_b200 import dense
    rng = np.random.default_rng(12)
    counts = []
    for t in range(3):
        Y = rng.standard_normal((300, 64)); X = rng.standard_normal((1, 64))
        xh, yh = C.stage_host(X), C.stage_host(Y)
        xs, ys = _dev(xh), _dev(yh)
        m = C.exact_row_margin(xs.norm16.item(), xs.err16.item(), ys.maxima[0].item(), ys.maxima[1].item(), 64)
        _, nc, cv = _fallback_rows(xs, ys, 10, 0.0, kc=10)
        assert nc[0] == 10
        B = C.add_ru(float(cv[0, 9]), m)
        fb_at, nc_at, cv_at = _fallback_rows(xs, ys, 10, B, kc=10)
        assert nc_at[0] == 10 and cv_at[0, 9] == cv[0, 9] and fb_at == []
        below = math.nextafter(B, -math.inf)
        fb_below, nc_below, _ = _fallback_rows(xs, ys, 10, below, kc=10)
        assert nc_below[0] == 10 and fb_below == [0]
        counts.append((len(fb_at), len(fb_below)))
        for thr in (B, below):
            oi, ov = O.exact_topk(xh.f64, yh.f64, 32, thr, normalized=True)
            for k in KS:
                i, v, _ = dense.dense_topk_exact(xs, ys, k, thr, k_cand=10 if k <= 10 else None)
                _same(i, v, oi[:, :k], ov[:, :k], ("B boundary", k, thr))
    print(f"certificate, thr = B / thr = B - ulp: fallback rows {counts}")


def test_certificate_kth_above_b_is_certified():
    rng = np.random.default_rng(13)
    Y = rng.standard_normal((2000, 64))
    X = rng.standard_normal((40, 64))
    for i in range(40):                                      # 4 planted close neighbours per row
        Y[4 * i:4 * i + 4] = X[i] + 0.1 * rng.standard_normal((4, 64))
    xh, yh = C.stage_host(X), C.stage_host(Y)
    fb, nc, cv = _fallback_rows(_dev(xh), _dev(yh), 4, 0.0)
    oi, ov = O.exact_topk(xh.f64, yh.f64, 4, 0.0, normalized=True)
    for i in range(40):                                      # the host restatement agrees that the k-th score beats B
        assert ov[i, 3] > C.add_ru(float(cv[i, -1]), xh.margin(i, yh))
    print(f"certificate, k-th > B: {len(fb)} fallback rows of 40")
    assert (nc == 16).all() and fb == []
    _exact_all(xh, yh, 0.0)
    _exact_all(xh, None, 0.0, self_match=True)


@pytest.mark.parametrize("tie", [True, False])
def test_certificate_tie_at_b(tie):
    from polyfuzz_b200 import dense
    xh, yh, info = C.tie_at_b(np.random.default_rng(1), tie=tie)
    xs, ys = _dev(xh), _dev(yh)
    fb, nc, cv = _fallback_rows(xs, ys, info["k"], 0.0, kc=info["kc"])
    assert nc[0] == info["kc"] and cv[0, -1] == info["s_kc"]
    print(f"certificate, k-th {'==' if tie else '>'} B: fallback rows {fb}")
    assert fb == ([0] if tie else [])
    oi, ov = O.exact_topk(xh.f64, yh.f64, 100, 0.0, normalized=True)
    i, v, _ = dense.dense_topk_exact(xs, ys, info["k"], 0.0, k_cand=info["kc"])
    _same(i, v, oi[:, :info["k"]], ov[:, :info["k"]], "tie")
    _exact_all(xh, yh, 0.0)


# ---- top_n > 32 --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("side", ["from", "to"])
def test_topn_keeps_eligible_rows_when_the_margin_exceeds_m_max(side):
    """The pair (0, 0) scores c > thr canonically but below t_f in the filter.  The bound pass has no k-th entry for row 0,
    so its threshold must be thr - M_i, not the filter's global cut."""
    from polyfuzz_b200 import dense
    xh, yh, X, Y, c, thr = C.broken_pair(64, 200, np.random.default_rng(5), side=side)
    xs, ys = _dev(xh), _dev(yh)
    for k in KS_TOPN:
        for sp in (None, 1):
            i, v, _ = dense.dense_topn_bounded(xs, ys, k, thr, n_splits=sp)
            assert i[0, 0].item() == 0 and v[0, 0].item() == c, (k, sp, i[0, :3].tolist())
    _exact_all(xh, yh, thr)
    for t in (c, math.nextafter(c, -math.inf), c - C.exact_margin_max(64) / 2, 0.0):
        _exact_all(xh, yh, t, ks=KS_TOPN)


@pytest.mark.parametrize("two_cta", ["0", "1"])
def test_off_norm_and_edge_rows_on_both_sides(two_cta, monkeypatch):
    monkeypatch.setenv("PFZ_K4_2CTA", two_cta)
    rng = np.random.default_rng(14)
    d = 64
    off = C.off_norm_rows(d)[0]
    base = rng.standard_normal((150, d))
    # subnormal dot(x, x), pointing roughly along base rows 0-2, so that they rank high against them
    sub = np.where(np.abs(base[:3]) > 1, 1.2, 0.75) * 2.0 ** -537 * np.sign(base[:3])
    X = np.vstack([off, sub, C.fp16_edge_rows(d, rng), C.aligned_rows(d, 4, rng), base[:40]])
    Y = np.vstack([base, off, sub, C.aligned_rows(d, 4, rng)])
    with np.errstate(over="ignore"):
        for a, b in ((X, Y), (Y, X)):
            ah, bh = C.stage_host(a), C.stage_host(b)
            for thr in (0.0, 0.05, -1.0):
                _exact_all(ah, bh, thr, splits=(None,))
        xh = C.stage_host(X)
        _exact_all(xh, None, 0.0, self_match=True, splits=(None,))
        # the staged rows of stage_exact, not the host image, give the same results
        from polyfuzz_b200 import dense
        xs, ys = dense.stage_exact(X), dense.stage_exact(Y)
        oi, ov = O.exact_topk(X, Y, 100, 0.0)
        for k in (10, 40, 100):
            i, v, _ = dense.dense_topk_exact(xs, ys, k, 0.0)
            _same(i, v, oi[:, :k], ov[:, :k], ("staged", k))


def test_embeddings_api_on_off_norm_rows():
    from polyfuzz_b200 import Embeddings, dense
    from polyfuzz_b200.distributed import merge_topk_any, shard_bounds
    from oracle.assemble import assemble
    rng = np.random.default_rng(15)
    d = 48
    off = C.off_norm_rows(d)[0]
    ef = np.vstack([off, rng.standard_normal((60, d))])
    et = np.vstack([rng.standard_normal((80, d)), off, off[:3] * -1.0])
    frm = [f"from {i}" for i in range(len(ef))]
    to = [f"to {i}" for i in range(len(et))]
    with np.errstate(over="ignore"):
        oi, ov = O.exact_topk(ef, et, 40, 0.0)
        df = Embeddings(min_similarity=0.0, top_n=40, precision="fp64").match(frm, to, ef, et)
    exp = assemble(frm, to, oi, ov)
    cells = lambda f, c: [None if (isinstance(v, float) and np.isnan(v)) else v for v in f[c].tolist()]   # noqa: E731
    assert list(df.columns) == list(exp.keys())
    for col in df.columns:
        assert cells(df, col) == cells(exp, col), col
    # from-rows 3 (dot(x, x) overflows: x~ = +-0) and 4 (zero) have no eligible to-row; row 6 (dot(x, x) underflows, so x~ = x
    # ~ 3e-300) has eligible ones, but their scores round to 0.000 and the frame blanks them
    assert (oi[3] < 0).all() and (oi[4] < 0).all() and (oi[6] >= 0).all() and 0 < ov[6, 0] < 1e-299
    assert [r for r, v in enumerate(cells(df, "To")) if v is None] == [3, 4, 6]
    xs = dense.stage_exact(ef)
    parts_i, parts_v = [], []
    for r in range(2):
        lo, hi = shard_bounds(len(et), 2, r)
        i, v, _ = dense.dense_topk_exact(xs, dense.stage_exact(et[lo:hi]), 40, 0.0, to_index_base=lo)
        parts_i.append(i); parts_v.append(v)
    mi, mv = merge_topk_any(torch.stack(parts_i), torch.stack(parts_v), 40)
    _same(mi, mv, oi, ov, "sharded")
