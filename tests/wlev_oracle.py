"""ctypes bindings to wlev_oracle.c, the CPU restatement of weighted Levenshtein (rapidfuzz.distance.Levenshtein with
weights = (insertion, deletion, substitution)) (TEST INFRASTRUCTURE, NOT PRODUCT CODE).  The library is compiled with gcc into a
temporary directory on first use, so nothing is written into the source tree."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

from dl_oracle import _pack, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "wlev_oracle.c")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        tmp = tempfile.mkdtemp(prefix="pfz_wlev_oracle_")
        try:
            so = os.path.join(tmp, "libwlev_oracle.so")
            env = dict(os.environ); env.pop("CC", None)
            subprocess.check_call(["gcc", "-O3", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra",
                                   "-shared", "-o", so, _SRC], env=env)
            L = ctypes.CDLL(so)                     # stays mapped after the file is removed
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
        vp, i32, i64, f64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_double
        L.oracle_wlev_matrix.argtypes = [vp, vp, i32, vp, vp, i32, i32, i32, i32, vp, vp, i32]
        L.oracle_wlev_matrix.restype = ctypes.c_int
        L.oracle_wlev_topk.argtypes = [vp, vp, i32, vp, vp, i32, i32, i32, i32, i32, f64, i32, i64, vp, vp, vp, i32]
        L.oracle_wlev_topk.restype = ctypes.c_int
        _LIB = L
    return _LIB


def _w(weights):
    return (1, 1, 1) if weights is None else tuple(int(x) for x in weights)


def wlev_matrix(from_list, to_list, weights, n_threads=1):
    """(D int64 [n_from, n_to], M int64 [n_from, n_to]): weighted distances and maxima."""
    fb, fo = _pack(from_list); tb, to = _pack(to_list)
    d = np.empty((len(from_list), len(to_list)), dtype=np.int64)
    mx = np.empty_like(d)
    lib().oracle_wlev_matrix(_p(fb), _p(fo), len(from_list), _p(tb), _p(to), len(to_list), *_w(weights), _p(d), _p(mx), int(n_threads))
    return d, mx


def wlev(a, b, weights):
    """(D, M) of one pair."""
    d, mx = wlev_matrix([a], [b], weights)
    return int(d[0, 0]), int(mx[0, 0])


def score_matrix(from_list, to_list, weights, n_threads=1):
    """float64 [n_from, n_to] of 1 - D/M (1 where M == 0), the kernel's expression."""
    d, mx = wlev_matrix(from_list, to_list, weights, n_threads)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(mx > 0, 1.0 - d.astype(np.float64) / mx.astype(np.float64), 1.0)


def wlev_topk(from_list, to_list, weights, k, score_cutoff=0.0, exclude_self=False, self_shift=0, n_threads=1):
    """Per from-row the k best to-indices (score desc, index asc; score >= score_cutoff), their scores and weighted distances:
    (idx int32 [n, k], score float64 [n, k], dist int64 [n, k]), empty slots (-1, 0.0, -1)."""
    fb, fo = _pack(from_list); tb, to = _pack(to_list)
    n = len(from_list)
    idx = np.empty((n, k), dtype=np.int32); sc = np.empty((n, k), dtype=np.float64); d = np.empty((n, k), dtype=np.int64)
    lib().oracle_wlev_topk(_p(fb), _p(fo), n, _p(tb), _p(to), len(to_list), *_w(weights), int(k), float(score_cutoff),
                           int(bool(exclude_self)), int(self_shift), _p(idx), _p(sc), _p(d), int(n_threads))
    return idx, sc, d


def wlev_argbest(from_list, to_list, weights, score_cutoff=0.0, exclude_self=False, self_shift=0, n_threads=1):
    """wlev_topk with k = 1, as [n] arrays."""
    i, s, d = wlev_topk(from_list, to_list, weights, 1, score_cutoff, exclude_self, self_shift, n_threads)
    return i[:, 0], s[:, 0], d[:, 0]


def norm_wlev(a, b, weights):
    """rapidfuzz's Levenshtein.normalized_similarity(a, b, weights=weights) as the oracle computes it."""
    return float(score_matrix([a], [b], weights)[0, 0])


def normalized_similarity(s1, s2, weights=None):
    """Stand-in for rapidfuzz.distance.Levenshtein.normalized_similarity, under the name the matchers' scorer resolution reads:
    partials of it are what users pass as scorer, and the reference's own EditDistance can call them."""
    return norm_wlev(s1, s2, weights)
