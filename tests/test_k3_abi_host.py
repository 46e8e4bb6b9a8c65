"""The argument rules of K3's and K3b's C entry points (pfz_lev_rows, pfz_fuzz_rows), CPU only: both check every combination of
metric or scorer, epilogue (k), source (cand_idx), matrix, gate and part_dist before any CUDA call, so a call with n_ids = 0
and null buffers returns 0 when the combination is allowed, and 1 with pfz_last_error() naming a broken rule when it is not."""
import ctypes
import itertools

import numpy as np

from polyfuzz_b200 import _lib

BUF = np.zeros(64, dtype=np.int64)          # a host address for the non-NULL pointers: nothing is read with n_ids = 0
NN = ctypes.c_void_p(BUF.ctypes.data)
TOPK_METRICS = (2, 3, 4, 5, 7, 9)           # NORM_LEV, RATIO, JARO, JARO_WINKLER, NORM_OSA, NORM_DL
# (cand_idx, n_splits, c, pos_of): all pairs, then candidate mode
SOURCES = [(None, 1, 0, None), (None, 3, 0, None), (None, 0, 0, None), (NN, 1, 4, NN), (NN, 2, 4, NN), (NN, 1, 0, NN),
           (NN, 1, 4, None)]


def _source_rules(cand, n_splits, c, pos_of):
    if cand is not None:
        return ["candidate mode"] if n_splits != 1 or c < 1 or pos_of is None else []
    return ["n_splits < 1"] if n_splits < 1 else []


def _k3_rules(metric, n_words, k, part_dist, matrix, gate, source):
    """The rules a pfz_lev_rows call breaks (substrings of their messages); [] = allowed."""
    broken = _source_rules(*source)
    if not 0 <= metric <= 9:
        broken.append("unknown metric")
    if n_words not in (0, 1, 2, 4, 8, 16):
        broken.append("n_words")
    if not 0 <= k <= 32:
        broken.append(f"k={k} unsupported")
    if k >= 1 and metric not in TOPK_METRICS:
        broken.append("top-k metric")
    if k >= 1 and (part_dist or matrix):
        broken.append("top-k has no distance output")
    if k == 0 and not part_dist:
        broken.append("arg-best needs part_dist")
    if matrix and metric in (4, 5):
        broken.append("not available for the Jaro metrics")
    if gate and metric not in (8, 9):
        broken.append("gate is for DL / NORM_DL only")
    if matrix and gate:
        broken.append("gate must be NULL with a matrix")
    return broken


def _check(name, rc, broken):
    msg = _lib.load().pfz_last_error().decode()
    if not broken:
        assert rc == 0, (name, msg)
    else:
        assert rc == 1 and any(b in msg for b in broken), (name, broken, msg)


def test_lev_rows_rules():
    lib = _lib.load()
    n_allowed = 0
    for metric, k, part_dist, matrix, gate, source in itertools.product(range(-1, 11), (-1, 0, 1, 5, 32, 33), (False, True),
                                                                         (False, True), (False, True), SOURCES):
        cand, n_splits, c, pos_of = source
        rc = lib.pfz_lev_rows(NN, NN, 10, NN, 0, 0, NN, NN, NN, NN, NN, 20, metric, 0.5, 0, 0, n_splits, k, cand, c, pos_of, NN, NN,
                              NN if part_dist else None, NN if matrix else None, 20 if matrix else 0, NN if gate else None, NN, None)
        broken = _k3_rules(metric, 0, k, part_dist, matrix, gate, source)
        _check(("pfz_lev_rows", metric, k, part_dist, matrix, gate, source), rc, broken)
        n_allowed += not broken
    assert n_allowed > 100
    for n_words in (-1, 0, 1, 2, 3, 4, 8, 16, 32):
        rc = lib.pfz_lev_rows(NN, NN, 10, NN, 0, n_words, NN, NN, NN, NN, NN, 20, 2, 0.5, 0, 0, 1, 0, None, 0, None, NN, NN, NN, None, 0,
                              None, NN, None)
        _check(("pfz_lev_rows", n_words), rc, _k3_rules(2, n_words, 0, True, False, False, SOURCES[0]))


def test_fuzz_rows_rules():
    lib = _lib.load()
    ptrs = (ctypes.c_void_p * 38)()
    for scorer, n_ptrs, n_words, k, source in itertools.product(range(-1, 11), (37, 38), (0, 1, 2, 3, 4, 8, 16), (-1, 0, 1, 32, 33),
                                                                SOURCES):
        cand, n_splits, c, pos_of = source
        rc = lib.pfz_fuzz_rows(ptrs, n_ptrs, 10, 0, n_words, 20, scorer, 50.0, 0, 0, n_splits, k, cand, c, pos_of, None)
        broken = _source_rules(*source)
        broken += ["expected 38 pointers"] if n_ptrs != 38 else []
        broken += ["unknown scorer"] if not 0 <= scorer <= 9 else []
        broken += ["n_words"] if n_words not in (1, 2, 4, 8, 16) else []
        broken += [f"k={k} unsupported"] if not 0 <= k <= 32 else []
        _check(("pfz_fuzz_rows", scorer, n_ptrs, n_words, k, source), rc, broken)

