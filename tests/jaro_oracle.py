"""ctypes bindings to jaro_oracle.c, the CPU restatement of jellyfish's Jaro / Jaro-Winkler similarity
(TEST INFRASTRUCTURE, NOT PRODUCT CODE).  The library is compiled with gcc into a temporary directory on first use,
so nothing is written into the source tree."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "jaro_oracle.c")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        tmp = tempfile.mkdtemp(prefix="pfz_jaro_oracle_")
        try:
            so = os.path.join(tmp, "libjaro_oracle.so")
            env = dict(os.environ); env.pop("CC", None)
            subprocess.check_call(["gcc", "-O3", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra",
                                   "-shared", "-o", so, _SRC], env=env)
            L = ctypes.CDLL(so)                     # stays mapped after the file is removed
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
        vp, i32, i64, f64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_double
        L.oracle_jaro_pair.argtypes = [vp, i32, vp, i32, i32, vp]
        L.oracle_jaro_pair.restype = f64
        L.oracle_jaro_argbest.argtypes = [vp, vp, i32, vp, vp, i32, i32, f64, i32, i64, vp, vp, vp, i32]
        L.oracle_jaro_argbest.restype = ctypes.c_int
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


def _u32(s):
    a = np.frombuffer(s.encode("utf-32-le", "surrogatepass"), dtype=np.uint32)
    return np.ascontiguousarray(a) if a.size else np.zeros(1, dtype=np.uint32)


def jaro_pair(s1, s2, winkler=True):
    """(score, match count m) of scorer(s1, s2) -- s1 is the from-string."""
    m = ctypes.c_int32(0)
    s = lib().oracle_jaro_pair(_p(_u32(s1)), len(s1), _p(_u32(s2)), len(s2), int(bool(winkler)), ctypes.byref(m))
    return s, m.value


def jaro_similarity(s1, s2):
    return jaro_pair(s1, s2, winkler=False)[0]


def jaro_winkler_similarity(s1, s2):
    return jaro_pair(s1, s2, winkler=True)[0]


def jaro_argbest(from_list, to_list, metric="jaro_winkler", score_cutoff=0.0, exclude_self=False, self_shift=0, n_threads=1):
    """Best to-index per from-row (first maximal score >= score_cutoff), its score and match count (-1 = none)."""
    assert metric in ("jaro", "jaro_winkler")
    fb, fo = _pack(from_list); tb, to = _pack(to_list)
    n = len(from_list)
    bi = np.empty(n, dtype=np.int32); bs = np.empty(n, dtype=np.float64); bd = np.empty(n, dtype=np.int32)
    lib().oracle_jaro_argbest(_p(fb), _p(fo), n, _p(tb), _p(to), len(to_list), int(metric == "jaro_winkler"), float(score_cutoff),
                              int(bool(exclude_self)), int(self_shift), _p(bi), _p(bs), _p(bd), int(n_threads))
    return bi, bs, bd
