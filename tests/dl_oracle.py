"""ctypes bindings to dl_oracle.c, the CPU restatement of unrestricted Damerau-Levenshtein (rapidfuzz.distance.DamerauLevenshtein,
Lowrance-Wagner with unit costs) (TEST INFRASTRUCTURE, NOT PRODUCT CODE).  The library is compiled with gcc into a temporary directory on first use, so nothing is
written into the source tree."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "dl_oracle.c")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        tmp = tempfile.mkdtemp(prefix="pfz_dl_oracle_")
        try:
            so = os.path.join(tmp, "libdl_oracle.so")
            env = dict(os.environ); env.pop("CC", None)
            subprocess.check_call(["gcc", "-O3", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra",
                                   "-shared", "-o", so, _SRC], env=env)
            L = ctypes.CDLL(so)                     # stays mapped after the file is removed
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
        vp, i32, i64, f64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_double
        L.oracle_dl_matrix.argtypes = [vp, vp, i32, vp, vp, i32, vp, i32]
        L.oracle_dl_matrix.restype = ctypes.c_int
        L.oracle_dl_argbest.argtypes = [vp, vp, i32, vp, vp, i32, i32, f64, i32, i64, vp, vp, vp, i32]
        L.oracle_dl_argbest.restype = ctypes.c_int
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _pack(strings):
    n = len(strings)
    offs = np.zeros(n + 1, dtype=np.int64)
    if n:
        np.cumsum(np.fromiter(map(len, strings), dtype=np.int64, count=n), out=offs[1:])
    blob = np.frombuffer("".join(strings).encode("utf-32-le", "surrogatepass"), dtype=np.uint32)
    if blob.size == 0:
        blob = np.zeros(1, dtype=np.uint32)
    return np.ascontiguousarray(blob), offs


def dl_matrix(from_list, to_list, n_threads=1):
    """int32 [n_from, n_to] DL distances."""
    fb, fo = _pack(from_list); tb, to = _pack(to_list)
    d = np.empty((len(from_list), len(to_list)), dtype=np.int32)
    lib().oracle_dl_matrix(_p(fb), _p(fo), len(from_list), _p(tb), _p(to), len(to_list), _p(d), int(n_threads))
    return d


def dl(a, b):
    return int(dl_matrix([a], [b])[0, 0])


def dl_argbest(from_list, to_list, metric="norm_dl", score_cutoff=0.0, exclude_self=False, self_shift=0, n_threads=1):
    """Best to-index per from-row (first maximal score, score >= score_cutoff for norm_dl; smallest distance for dl), its
    score (norm_dl, or -distance) and DL distance (-1 = none)."""
    assert metric in ("dl", "norm_dl")
    fb, fo = _pack(from_list); tb, to = _pack(to_list)
    n = len(from_list)
    bi = np.empty(n, dtype=np.int32); bs = np.empty(n, dtype=np.float64); bd = np.empty(n, dtype=np.int32)
    lib().oracle_dl_argbest(_p(fb), _p(fo), n, _p(tb), _p(to), len(to_list), int(metric == "norm_dl"), float(score_cutoff),
                             int(bool(exclude_self)), int(self_shift), _p(bi), _p(bs), _p(bd), int(n_threads))
    return bi, bs, bd


def norm_dl(a, b):
    return float(dl_argbest([a], [b], "norm_dl", score_cutoff=float("-inf"))[1][0])
