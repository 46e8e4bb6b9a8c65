"""Score cutoffs that land on achieved scores (TEST INFRASTRUCTURE, NOT PRODUCT CODE): the cutoff grid, the (|a|, |b|, LCS)
triples of fuzz.ratio, and a seeded generator of the pairs where rapidfuzz's two cutoff steps disagree.

rapidfuzz applies a cutoff c of the 0..100 scorers in two steps: fuzz.ratio keeps ns = 1 - indel/(|a|+|b|) only if
ns >= c/100 and returns ns*100, partial_ratio scores its windows at c/100; then the caller keeps the result only if it is
>= c.  The steps disagree whenever (ns*100)/100 != ns in doubles: for such a pair, a cutoff equal to its own score rejects it
(a "boundary pair").  oracle/fuzz.py restates both steps."""
import math

import numpy as np

from oracle import fuzz as ofuzz


def cutoff_grid():
    """u*100 for u in {k/100} and {k/1000}, ascending, duplicates removed."""
    return sorted({(k / 100) * 100 for k in range(101)} | {(k / 1000) * 100 for k in range(1001)})


def neighbours(c):
    """c and the doubles just below and above it."""
    return (math.nextafter(c, -math.inf), c, math.nextafter(c, math.inf))


def ratio_ns(la, lb, lcs):
    m = la + lb
    return 1.0 - (m - 2 * lcs) / m if m else 1.0


def is_boundary_score(ns):
    """fuzz.ratio's score ns*100 at a cutoff equal to itself is rejected by the c/100 step"""
    return not ns >= (ns * 100.0) / 100.0


def ratio_strings(la, lb, lcs, x="a", y="b", z="c"):
    """A pair with |a| = la, |b| = lb and LCS(a, b) = lcs (x shared, y only in a, z only in b)."""
    return x * lcs + y * (la - lcs), x * lcs + z * (lb - lcs)


def ratio_triples(max_len=60):
    """Every (|a|, |b|, lcs) with lengths 1..max_len."""
    return [(la, lb, l) for la in range(1, max_len + 1) for lb in range(1, max_len + 1) for l in range(min(la, lb) + 1)]


def wratio_row(args):
    """[WRatio(a, b) for b in to] at cutoff 0 with the C LCS (a process-pool worker: the pool's processes import this module
    afresh, so the swap of oracle.fuzz.lcs_len is made here)."""
    import lcs_oracle
    a, to = args
    ofuzz.lcs_len = lcs_oracle.lcs_len
    return [ofuzz.WRatio(a, b) for b in to]


def boundary_pairs(scorer, n, seed, alphabet="abc ", lo=1, hi=32, max_tries=200000):
    """n random pairs (a, b, s) over `alphabet` where scorer(a, b, 0) == s > 0 but scorer(a, b, s) == 0: the cutoff equal to
    the achieved score rejects the pair."""
    fn = ofuzz.SCORERS[scorer]
    rng = np.random.default_rng(seed)
    chars = list(alphabet)
    out = []
    for _ in range(max_tries):
        la, lb = rng.integers(lo, hi + 1, 2)
        a = "".join(rng.choice(chars, la)); b = "".join(rng.choice(chars, lb))
        s = fn(a, b, 0)
        if s > 0 and fn(a, b, s) == 0:
            out.append((a, b, s))
            if len(out) == n:
                break
    return out
