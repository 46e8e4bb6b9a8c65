"""Inputs that attack the exactness argument of the Embeddings exact mode (precision="fp64", DESIGN.md 4.6 and 4.7), and the
host restatement of the bounds it rests on.

The exact mode is exact because of an error bound, not because of its fp64 arithmetic: an fp16 tensor-core filter picks the
candidates, and a margin (M_i per row, M_max a priori, gamma = d_pad 2^-22 for the fp32 accumulation) decides whether a row
is certified or goes to brute force.  Gaussian rows exercise little of that: their fp16 rounding errors cancel, their norms
are 1 to an ulp and their thresholds sit far from the filter's cut.  The constructors below aim at the edges instead:

  aligned_rows         x~ components just below fp16 midpoints just above powers of two, one sign pattern for the from-
                       and to-rows: every rounding error is ~2^-11 relative and they add up (x^.y^ - x~.y~ ~ 0.95 M_max);
  off_norm_rows        dot(x, x) subnormal, so ||x~|| is far from 1 (0.75 and 1.2), overflowing rows (x~ = +-0), zero
                       rows, single non-zero entries (one of them so small that dot(x, x) underflows to 0);
  fp16_edge_rows       x~ entries that are exact fp16 ties, fp16 subnormals, +-2^-25 and its neighbours, -0.0;
  same_sign_f16        positive fp16 rows with full 11-bit mantissas: every fp32 addition rounds, nothing cancels;
  margin_thresholds    thresholds at, next to and inside the margin of one pair;
  broken_pair          staged rows (the ExactRows contract, honest bounds) whose fp16 side is pushed along y~ by
                       several 2^-11: M_i > M_max and f < t_f < thr < c, deterministically;
  tie_at_b             hand-staged rows whose certificate bound B = s_k' + M_i equals the exact k-th score, bit for bit.

Restated from csrc/pfz_dense.cu with the same constant expressions: exact_gamma, exact_margin_max, exact_row_margin (every
operation rounded up, as the kernel's __d*_ru intrinsics), filter_threshold, and the exact row threshold of the top_n > 32
bound pass.  The staging is simulated with dense_exact_oracle.canon_normalize and numpy's float16 cast, which rounds to
nearest even straight from double, as __double2half does."""
import math
from fractions import Fraction

import numpy as np

import dense_exact_oracle as O

INF = math.inf


# ---- bounds (csrc/pfz_dense.cu) ----------------------------------------------------------------------------------------

def exact_gamma(d_pad):
    return d_pad * 2.0 ** -22


def exact_margin_max(d_pad):
    r = 1.0 + d_pad * 2.0 ** -50
    e = 2.0 ** -11 * r + 2.0 ** -25 * math.sqrt(float(d_pad))
    n = r + e
    m = 2.0 * e * n + e * e + exact_gamma(d_pad) * n * n + 2.0 * d_pad * 2.0 ** -53 * (n + e) * (n + e)
    return m * (1.0 + 2.0 ** -20)


def ru(q):
    """The double nearest above the exact rational q (q itself when representable)."""
    f = float(q)
    return f if Fraction(f) >= q else math.nextafter(f, INF)


def rd(q):
    f = float(q)
    return f if Fraction(f) <= q else math.nextafter(f, -INF)


def mul_ru(a, b):
    return ru(Fraction(a) * Fraction(b))


def add_ru(a, b):
    return ru(Fraction(a) + Fraction(b))


def exact_row_margin(nx, ex, Ny, Ey, d_pad):
    """M_i of a from-row: an upper bound on |fp32 filter score - canonical score| against every to-row."""
    g = exact_gamma(d_pad)
    m = mul_ru(ex, Ny)
    m = add_ru(m, mul_ru(nx, Ey))
    m = add_ru(m, mul_ru(ex, Ey))
    m = add_ru(m, mul_ru(mul_ru(g, nx), Ny))
    m = add_ru(m, mul_ru(mul_ru(2.0 * d_pad * 2.0 ** -53, add_ru(nx, ex)), add_ru(Ny, Ey)))
    return m


def filter_threshold(thr, d_pad):
    """t_f: the largest float <= thr - M_max(d_pad)."""
    t = math.nextafter(thr - exact_margin_max(d_pad), -INF)
    tf = np.float32(t)
    if float(tf) > t:
        tf = np.nextafter(tf, np.float32(-np.inf))
    return float(tf)


def f32_rd(x):
    """The largest float <= the double x."""
    f = np.float32(x)
    if float(f) > x:
        f = np.nextafter(f, np.float32(-np.inf))
    return float(f)


def exact_row_threshold(lo, m):
    """Row threshold of the exact top_n > 32 threshold pass for a lower bound `lo` of the canonical scores it must keep."""
    return f32_rd(rd(Fraction(lo) - Fraction(m)))


# ---- staging on the host -------------------------------------------------------------------------------------------------

def d_pad_of(d):
    return max(8, (d + 7) // 8 * 8)


def sq_norm(v):
    """||v||^2 as an exact rational (v: any float array)."""
    return sum((Fraction(float(a)) ** 2 for a in np.asarray(v, dtype=np.float64).ravel() if a != 0), Fraction(0))


def norm_ru(v):
    """An upper bound of ||v||, at most an ulp or two above it."""
    s = sq_norm(v)
    if s == 0:
        return 0.0
    e = (s.numerator.bit_length() - s.denominator.bit_length()) // 2  # sqrt of s / 4^e ~ 1, then scaled back exactly
    r = math.ldexp(math.sqrt(float(s / Fraction(4) ** e)), e)
    while Fraction(r) ** 2 < s:
        r = math.nextafter(r, INF)
    return r


class HostRows:
    """The host image of dense.ExactRows: f64, f16 (numpy, [n, d_pad]), norm16, err16 (float64[n]) and maxima."""

    def __init__(self, f64, f16, norm16=None, err16=None):
        self.f64 = np.asarray(f64, dtype=np.float64)
        self.f16 = np.asarray(f16, dtype=np.float16)
        h = self.f16.astype(np.float64)
        self.norm16 = np.array([norm_ru(r) for r in h]) if norm16 is None else np.asarray(norm16, dtype=np.float64)
        self.err16 = np.array([norm_ru(a - b) for a, b in zip(self.f64, h)]) if err16 is None else np.asarray(err16, np.float64)
        self.maxima = np.array([self.norm16.max(initial=0.0), self.err16.max(initial=0.0)])

    @property
    def d_pad(self):
        return self.f64.shape[1]

    def margin(self, i, other):
        """M_i of row i against the to-rows `other`."""
        return exact_row_margin(self.norm16[i], self.err16[i], other.maxima[0], other.maxima[1], self.d_pad)


def stage_host(X):
    """What stage_exact must produce for X: canonical rows, their fp16 rounding, honest bounds."""
    X = np.asarray(X, dtype=np.float64)
    n, d = X.shape
    f64 = np.zeros((n, d_pad_of(d)))
    f64[:, :d] = O.canon_normalize(X)
    return HostRows(f64, f64.astype(np.float16))


def f16_dot_exact(xh, yh):
    """Exact x^ . y^ of fp16 rows as integers in units of 2^-48 (every fp16 value is a multiple of 2^-24)."""
    a = (np.asarray(xh, dtype=np.float64) * 2.0 ** 24).astype(np.int64)
    b = (np.asarray(yh, dtype=np.float64) * 2.0 ** 24).astype(np.int64)
    return [[sum(int(p) * int(q) for p, q in zip(ra, rb)) for rb in b] for ra in a]


def f16_dot_fraction(xh, yh):
    return Fraction(f16_dot_exact(xh[None], yh[None])[0][0], 2 ** 48)


def canon_score(x64, y64):
    return float(O.canon_dot(np.asarray(x64)[None], np.asarray(y64)[None])[0, 0])


# ---- constructors ------------------------------------------------------------------------------------------------------

A_BELOW = 0.99 * 2.0 ** -11          # relative position of an aligned value: 1 % below the fp16 midpoint above 2^e


def aligned_rows(d, n, rng, signs=None):
    """n rows of width d whose canonical x~ has every component but one at +-2^e (1 + 0.99 2^-11): just below the fp16
    midpoint above a power of two, so fp16 rounds each of them down by ~2^-11 of its size.  Component 0 takes the rest of
    the unit norm.  All rows share the sign pattern `signs` (random when None) and place the exponents in random order."""
    if signs is None:
        signs = rng.choice([-1.0, 1.0], size=d)
    e0 = math.ceil(math.log2(1.0 / math.sqrt(d)))                     # two levels, 2^e0 and 2^(e0 - 1), fill the unit norm
    f = (1.0 + A_BELOW) ** 2
    n_hi = d - 1
    while n_hi * 4.0 ** e0 * f + (d - 1 - n_hi) * 4.0 ** (e0 - 1) * f >= 1.0 - 4.0 ** (e0 - 2):
        n_hi -= 1
    mags = np.array([2.0 ** e0] * n_hi + [2.0 ** (e0 - 1)] * (d - 1 - n_hi)) * (1.0 + A_BELOW)
    out = np.empty((n, d))
    for r in range(n):
        m = rng.permutation(mags)
        out[r, 1:] = m
        out[r, 0] = math.sqrt(1.0 - float(np.sum(m * m)))
    return out * signs


def off_norm_rows(d):
    """Rows whose staged norm is not 1, or that normalise degenerately.  Returns (X, labels)."""
    rows, labels = [], []
    t = 2.0 ** -537                   # (c t)^2 = c^2 subnormal ulps, rounded to one ulp for 0.71 < c < 1.22
    for c, lab in ((1.2, "subnormal dot, ||x~|| ~ 1.2"), (0.75, "subnormal dot, ||x~|| ~ 0.75")):
        r = np.full(d, c * t); r[1::2] *= -1.0
        rows.append(r); labels.append(lab)
    r = np.full(d, 1.2 * t); r[::3] = 0.8 * t                           # mixed: entries both above and below one ulp
    rows.append(r); labels.append("subnormal dot, mixed")
    r = np.zeros(d); r[:3] = [1e200, -3e200, 2e200]
    rows.append(r); labels.append("dot(x, x) overflows: x~ = +-0")
    rows.append(np.zeros(d)); labels.append("zero row")
    r = np.zeros(d); r[d // 2] = -5.0
    rows.append(r); labels.append("one non-zero entry")
    r = np.zeros(d); r[d - 1] = 3e-300
    rows.append(r); labels.append("one entry whose square underflows: x~ = x")
    return np.array(rows), labels


def _four_squares(r):
    """Non-negative integers (a, b, c, e) with a^2 + b^2 + c^2 + e^2 = r, the first as large as possible."""
    for a in range(math.isqrt(r), -1, -1):
        r1 = r - a * a
        for b in range(math.isqrt(r1), -1, -1):
            r2 = r1 - b * b
            if 2 * b * b < r2:
                break
            for c in range(math.isqrt(r2), -1, -1):
                e2 = r2 - c * c
                if 2 * c * c < e2:
                    break
                e = math.isqrt(e2)
                if e * e == e2:
                    return a, b, c, e
    raise AssertionError(r)


FP16_EDGE_UNITS = {                     # x~ entries in units of 2^-26 (exact doubles) and what fp16 makes of them
    "tie, rounds down to even": 2049 * 2 ** 12,          # 1024.5 fp16 ulps of [2^-3, 2^-2): rounds to 1024
    "tie, rounds up to even": 2051 * 2 ** 12,            # 1025.5 ulps: rounds to 1026
    "fp16 subnormal tie, rounds to even": 4 * 37 + 2,
    "fp16 subnormal": 4 * 101,
    "just below 2^-25": 1,
    "at 2^-25": 2,
    "just above 2^-25": 3,
    "fp16 subnormal, negative": -4 * 7,
    "at -2^-25": -2,
    "-2^-26, to -0": -1,
}


def fp16_edge_rows(d, rng, n=4):
    """Rows whose canonical x~ is exactly n_c 2^-26 with the FP16_EDGE_UNITS values placed in it: sum n_c^2 = 2^52, so
    dot(x, x) = 1 exactly, sqrt is exact and x~ = x.  Four filler components carry the rest of the norm; one entry is -0.0."""
    assert d >= len(FP16_EDGE_UNITS) + 5
    out = np.zeros((n, d))
    for r in range(n):
        pos = rng.permutation(d)
        vals = list(FP16_EDGE_UNITS.values())
        rest = 2 ** 52 - sum(v * v for v in vals)
        fill = _four_squares(rest)
        row = np.zeros(d)
        for p, v in zip(pos, vals + [s * f for s, f in zip(rng.choice([-1, 1], 4), fill)]):
            row[p] = v * 2.0 ** -26
        row[pos[len(vals) + 4]] = -0.0
        out[r] = row
    return out


def same_sign_f16(d, n, rng):
    """Positive fp16 rows with full 11-bit significands (the last significand bit set), all in [2^-7, 2^-4) x (1 .. 2)."""
    e = rng.integers(-7, -4, size=(n, d)).astype(np.float64)
    m = 1024 + 2 * rng.integers(0, 512, size=(n, d)) + 1                # odd: 11 significant bits
    return (m / 1024.0 * 2.0 ** e).astype(np.float16)


def margin_thresholds(c, f16, gamma_term, d_pad):
    """Thresholds for a pair with canonical score c and exact fp16 product f16 (a Fraction): c, c +- 1 ulp, c - M_max / 2,
    and a `drop` threshold whose t_f lies in [f16 + gamma ||x^|| ||y^||, c): a filter that obeys gamma must drop the pair."""
    mm = exact_margin_max(d_pad)
    out = {"c": c, "c + ulp": math.nextafter(c, INF), "c - ulp": math.nextafter(c, -INF), "c - M_max/2": c - mm / 2}
    lo = f16 + Fraction(gamma_term)
    thr = float(lo) + mm
    while Fraction(filter_threshold(thr, d_pad)) < lo:
        thr += 2.0 ** -26
    out["drop"] = thr
    return out


def broken_pair(d, n_to, rng, push=8, side="from"):
    """Staged rows that keep every ExactRows contract (f64 canonical, norm16 >= ||f16||, err16 >= ||f64 - f16||) but whose
    fp16 side is pushed along the partner row by `push` 2^-11, so that M_i > M_max.

    Row 0 of the from-side is y_0 plus a little noise, so (0, 0) is its best pair, with canonical score c.  side="from": the
    from-row's f16 is fp16(x~_0 - push 2^-11 y~_0), which raises e_x of that row; side="to": y_0's f16 is pushed along x~_0,
    which raises E_y and so M_i of every from-row.  Returns (xs, ys, X, Y, c, thr) with thr = c - M_max / 2, for which the
    pair is eligible (c > thr) while its exact fp16 product plus the gamma term stays at or below t_f(thr)."""
    Y = rng.standard_normal((n_to, d))
    X = np.vstack([Y[:1] + 0.05 * rng.standard_normal((1, d)), rng.standard_normal((3, d))])
    xs, ys = stage_host(X), stage_host(Y)
    delta = push * 2.0 ** -11
    if side == "from":
        f16 = xs.f16.copy(); f16[0] = (xs.f64[0] - delta * ys.f64[0]).astype(np.float16)
        xs = HostRows(xs.f64, f16)
    else:
        f16 = ys.f16.copy(); f16[0] = (ys.f64[0] - delta * xs.f64[0]).astype(np.float16)
        ys = HostRows(ys.f64, f16)
    c = canon_score(xs.f64[0], ys.f64[0])
    thr = c - exact_margin_max(xs.d_pad) / 2
    return xs, ys, X, Y, c, thr


def tie_at_b(rng, d=64, n_to=200, k=4, kc=10, tie=True):
    """One from-row and n_to to-rows, hand-staged so that the certificate bound B = s_kc + M_i (rounded up) equals the exact
    k-th score of the row (tie=True: the certificate must refuse it, a to-row scoring exactly B could tie) or lies one step
    below it (tie=False: certified).  The fp16 sides are multiples of 2^-8, so every fp32 filter score is exact and s_kc
    is known on the host; e_x (an upper bound, honest but inflated) tunes M_i.  Returns (xs, ys, info)."""
    q = 2.0 ** -8
    for _ in range(50):                                                 # B may step over the k-th score: draw again
        Y = rng.standard_normal((n_to, d))
        x = rng.standard_normal(d)
        for j in range(k):                                              # k close neighbours with distinct scores
            Y[j] = x + (0.15 + 0.05 * j) * rng.standard_normal(d)
        yn = O.canon_normalize(Y); xn = O.canon_normalize(x[None])
        y16 = (np.round(yn / q) * q).astype(np.float16)
        x16 = (np.round(xn / q) * q).astype(np.float16)
        ys = HostRows(yn, y16)
        xs0 = HostRows(xn, x16)
        f = [Fraction(v, 2 ** 48) for v in f16_dot_exact(x16, y16)[0]]
        s_kc = sorted(f, reverse=True)[kc - 1]
        assert Fraction(float(np.float32(float(s_kc)))) == s_kc        # an fp32 value: the filter's kc-th score is exact
        s_kc = float(s_kc)
        ck = float(np.sort(O.canon_dot(xn, yn)[0])[::-1][k - 1])
        nx = xs0.norm16[0]
        Ny, Ey = ys.maxima

        def b_of(ex):
            return add_ru(s_kc, exact_row_margin(nx, ex, Ny, Ey, d))

        lo, hi = xs0.err16[0], 1.0                                      # B(lo) < ck <= B(hi); B is monotone in e_x
        assert b_of(lo) < ck <= b_of(hi), (b_of(lo), ck)
        while True:
            mid = lo + (hi - lo) / 2
            if mid in (lo, hi):
                break
            lo, hi = (mid, hi) if b_of(mid) < ck else (lo, mid)
        if tie and b_of(hi) != ck:
            continue
        ex = hi if tie else lo
        xs = HostRows(xn, x16, norm16=[nx], err16=[ex])
        return xs, ys, dict(B=b_of(ex), ck=ck, s_kc=s_kc, k=k, kc=kc, margin=exact_row_margin(nx, ex, Ny, Ey, d), x=xn, y=yn)
    raise AssertionError("no draw put B exactly on the k-th score")
