"""CPU checks that every input of tests/dense_cert_cases.py has the property it was built for, using the restated bounds and
exact products of the fp16 rows.  Without them a passing GPU test (tests/test_gpu_dense_exact_cert.py) would not show that
the hard branch of the exact mode's certificate or bound was reached."""
import math
import os
import sys
from fractions import Fraction

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dense_cert_cases as C                                          # noqa: E402
import dense_exact_oracle as O                                        # noqa: E402


def test_restated_bounds_keep_their_order():
    for d_pad in (8, 64, 768, 4096):
        mm = C.exact_margin_max(d_pad)
        r = 1.0 + d_pad * 2.0 ** -50
        e = 2.0 ** -11 * r + 2.0 ** -25 * math.sqrt(d_pad)
        # a row that meets the a-priori assumptions has M_i <= M_max
        assert C.exact_row_margin(r + e, e, r + e, e, d_pad) <= mm
        for thr in (0.0, 0.05, 0.5, -1.0):
            tf = C.filter_threshold(thr, d_pad)
            assert float(np.float32(tf)) == tf and Fraction(tf) < Fraction(thr) - Fraction(mm)
            assert float(np.nextafter(np.float32(tf), np.float32(np.inf))) > thr - mm - 2.0 ** -30
    assert 1.1e-3 < C.exact_margin_max(768) < 1.3e-3                  # DESIGN 4.6 quotes 1.2e-3 at d = 768


@pytest.mark.parametrize("d", [8, 64, 768, 4096])
def test_aligned_rows_round_the_same_way(d):
    X = C.aligned_rows(d, 2, np.random.default_rng(d))
    xs = C.stage_host(X)
    d_pad = xs.d_pad
    h = xs.f16.astype(np.float64)
    err = xs.f64 - h
    # every component but component 0 rounds towards zero by more than 0.98 2^-11 of its size
    rel = np.abs(err[:, 1:d]) / np.abs(xs.f64[:, 1:d])
    assert (rel > 0.98 * 2.0 ** -11).all() and (np.sign(err[:, 1:d]) == np.sign(xs.f64[:, 1:d])).all()
    assert (np.sign(xs.f64[0]) == np.sign(xs.f64[1])).all()
    c = C.canon_score(xs.f64[0], xs.f64[0])
    gap = Fraction(c) - C.f16_dot_fraction(xs.f16[0], xs.f16[0])
    mm, g = C.exact_margin_max(d_pad), C.exact_gamma(d_pad)
    # x^.y^ - x~.y~ nearly reaches the part of M_max that is not the accumulation term
    assert float(gap) > 0.75 * (mm - 1.01 * g), float(gap) / mm
    assert float(gap) <= xs.margin(0, xs)


def test_off_norm_rows():
    d = 32
    X, labels = C.off_norm_rows(d)
    xs = C.stage_host(X)
    d_pad = xs.d_pad
    norms = [math.sqrt(float(C.sq_norm(r))) for r in xs.f64]
    big = 1.0 + d_pad * 2.0 ** -50
    assert norms[0] > big and norms[0] > 1.19 and norms[2] > big     # above the ||x~|| <= 1 + d_pad 2^-50 of M_max
    assert norms[1] < 0.76
    ss = O.canon_self_dot(X)
    assert 0 < ss[0] < 2.0 ** -1022 and 0 < ss[1] < 2.0 ** -1022       # subnormal dot(x, x)
    with np.errstate(over="ignore"):
        assert np.isinf(O.canon_self_dot(X[3:4]))[0]
    assert (xs.f64[3] == 0).all() and np.signbit(xs.f64[3, 1])         # x / inf: -0.0 where x < 0
    assert (xs.f64[4] == 0).all() and not np.signbit(xs.f64[4]).any()
    assert xs.f64[5, d // 2] == -1.0 and np.count_nonzero(xs.f64[5]) == 1
    assert ss[6] == 0 and xs.f64[6, d - 1] == 3e-300 and xs.f16[6, d - 1] == 0   # not normalised: dot(x, x) underflows
    # as to-rows they raise N_y above the n = r + e that M_max assumes
    e = 2.0 ** -11 * big + 2.0 ** -25 * math.sqrt(d_pad)
    assert xs.maxima[0] > big + e
    assert len(labels) == len(X)


def test_fp16_edge_rows_stage_to_the_intended_values():
    d = 40
    E = C.fp16_edge_rows(d, np.random.default_rng(0))
    assert (O.canon_self_dot(E) == 1.0).all() and np.array_equal(O.canon_normalize(E), E)
    units = C.FP16_EDGE_UNITS
    want = {"tie, rounds down to even": 1024 * 2.0 ** -13, "tie, rounds up to even": 1026 * 2.0 ** -13,
            "fp16 subnormal tie, rounds to even": 38 * 2.0 ** -24, "fp16 subnormal": 101 * 2.0 ** -24,
            "just below 2^-25": 0.0, "at 2^-25": 0.0, "just above 2^-25": 2.0 ** -24,
            "fp16 subnormal, negative": -7 * 2.0 ** -24, "at -2^-25": -0.0, "-2^-26, to -0": -0.0}
    for row in E:
        h = row.astype(np.float16)
        for name, u in units.items():
            p = np.nonzero(row == u * 2.0 ** -26)[0]
            assert len(p) == 1, name
            assert h[p[0]] == want[name] and np.signbit(h[p[0]]) == np.signbit(want[name]), name
        assert np.signbit(row[row == 0]).sum() == 1                      # one -0.0 entry


@pytest.mark.parametrize("d", [8, 64, 768, 4096])
def test_same_sign_rows_have_full_mantissas(d):
    h = C.same_sign_f16(d, 3, np.random.default_rng(d))
    bits = h.view(np.uint16)
    assert (h > 0).all() and ((bits & 1) == 1).all() and ((bits >> 10) & 0x1F).min() > 0


def test_margin_thresholds_inside_the_margin():
    X = C.aligned_rows(64, 1, np.random.default_rng(7))
    xs = C.stage_host(X)
    c = C.canon_score(xs.f64[0], xs.f64[0])
    f16 = C.f16_dot_fraction(xs.f16[0], xs.f16[0])
    gterm = C.mul_ru(C.exact_gamma(64), C.mul_ru(xs.norm16[0], xs.norm16[0]))
    t = C.margin_thresholds(c, f16, gterm, 64)
    assert t["c - ulp"] < t["c"] < t["c + ulp"] and t["c - M_max/2"] < c
    tf = Fraction(C.filter_threshold(t["drop"], 64))
    assert f16 + Fraction(gterm) <= tf < Fraction(c)                   # a filter that obeys gamma drops the pair


@pytest.mark.parametrize("side", ["from", "to"])
def test_broken_pair_breaks_the_a_priori_margin(side):
    xs, ys, X, Y, c, thr = C.broken_pair(64, 200, np.random.default_rng(5), side=side)
    d_pad = xs.d_pad
    # the ExactRows contract: f64 canonical, honest bounds
    assert np.array_equal(xs.f64[:, :64], O.canon_normalize(X)) and np.array_equal(ys.f64[:, :64], O.canon_normalize(Y))
    for rows in (xs, ys):
        h = rows.f16.astype(np.float64)
        for i in range(len(h)):
            assert Fraction(rows.norm16[i]) ** 2 >= C.sq_norm(h[i]) and Fraction(rows.err16[i]) ** 2 >= C.sq_norm(rows.f64[i] - h[i])
    m = xs.margin(0, ys)
    assert m > C.exact_margin_max(d_pad)
    f16 = C.f16_dot_fraction(xs.f16[0], ys.f16[0])
    gterm = Fraction(C.exact_gamma(d_pad)) * Fraction(xs.norm16[0]) * Fraction(ys.maxima[0])
    tf = Fraction(C.filter_threshold(thr, d_pad))
    assert f16 + gterm <= tf < Fraction(thr) < Fraction(c)            # eligible, yet every filter that obeys gamma drops it
    assert abs(Fraction(c) - f16) <= Fraction(m)                      # ... while M_i still bounds the error
    # the fixed exact row threshold keeps it: f >= thr - M_i, rounded down, for any f within gamma of f16
    assert Fraction(C.exact_row_threshold(thr, m)) <= f16 - gterm
    # the canonical top-1 of from-row 0 is to-row 0, alone above thr
    oi, ov = O.exact_topk(xs.f64, ys.f64, 3, thr, normalized=True)
    assert oi[0].tolist() == [0, -1, -1] and ov[0, 0] == c


@pytest.mark.parametrize("tie", [True, False])
def test_tie_at_b(tie):
    xs, ys, info = C.tie_at_b(np.random.default_rng(1), tie=tie)
    assert (info["B"] == info["ck"]) == tie and info["B"] <= info["ck"]
    h = xs.f16.astype(np.float64)
    assert Fraction(xs.err16[0]) ** 2 >= C.sq_norm(xs.f64[0] - h[0]) and Fraction(xs.norm16[0]) ** 2 >= C.sq_norm(h[0])
    assert info["B"] > 0.0                                             # not certified by B <= thr (thr = 0)
    f = sorted((Fraction(v, 2 ** 48) for v in C.f16_dot_exact(xs.f16, ys.f16)[0]), reverse=True)
    assert float(f[info["kc"] - 1]) == info["s_kc"] > C.filter_threshold(0.0, xs.d_pad)
