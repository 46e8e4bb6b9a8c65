"""ctypes binding to lcs_oracle.c, a textbook C LCS with the semantics of oracle/fuzz.py's lcs_len (TEST INFRASTRUCTURE, NOT
PRODUCT CODE).  The library is compiled with gcc into a temporary directory on first use, so nothing is written into the
source tree.  tests/test_gpu_fuzz_long.py swaps it in for oracle.fuzz.lcs_len: on strings of a thousand code points
partial_ratio's one LCS per window would take the pure-Python DP hours."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "lcs_oracle.c")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        tmp = tempfile.mkdtemp(prefix="pfz_lcs_oracle_")
        try:
            so = os.path.join(tmp, "liblcs_oracle.so")
            env = dict(os.environ); env.pop("CC", None)
            subprocess.check_call(["gcc", "-O3", "-fPIC", "-Wall", "-Wextra", "-shared", "-o", so, _SRC], env=env)
            L = ctypes.CDLL(so)                     # stays mapped after the file is removed
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
        L.oracle_lcs.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64]
        L.oracle_lcs.restype = ctypes.c_int64
        _LIB = L
    return _LIB


def _u32(s):
    return np.frombuffer(s.encode("utf-32-le", "surrogatepass"), dtype=np.uint32)


def lcs_len(a, b):
    """Longest common subsequence length of two str (code points), as oracle.fuzz.lcs_len."""
    if not a or not b:
        return 0
    x, y = _u32(a), _u32(b)
    r = lib().oracle_lcs(x.ctypes.data, len(x), y.ctypes.data, len(y))
    if r < 0:
        raise MemoryError("oracle_lcs: allocation failed")
    return int(r)
