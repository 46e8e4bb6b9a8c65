"""Result assembly shared by the matchers -- the tail of polyfuzz/models/_utils.py:104-125, built
column-wise from the top-k arrays instead of through a (1+2k) x n unicode ndarray.

The string columns are gathered with Arrow (`take` on one Arrow array of the to_list, one thread per
column, GIL released) and handed to pandas as its native `str` columns -- the dtype the reference's
frame has under pandas 3 -- without per-element Python work or dtype inference."""
from concurrent.futures import ThreadPoolExecutor
from typing import List, Optional

import numpy as np
import pandas as pd

try:
    import pyarrow as pa
except Exception:                                        # pragma: no cover
    pa = None

_POOL = None


def _pool():
    global _POOL
    if _POOL is None:
        import os
        _POOL = ThreadPoolExecutor(max_workers=max(4, min(32, (os.cpu_count() or 8) // 2)), thread_name_prefix="pfz-assemble")
    return _POOL


def clip_top_n(top_n: int, to_list: Optional[List[str]]) -> int:
    """polyfuzz/models/_utils.py:54-56 -- only when a to_list is given."""
    if to_list is not None:
        top_n = min(top_n, len(set(to_list)))
    return top_n


def _str_dtype():
    try:
        dt = pd.StringDtype(na_value=np.nan)
        if pa is not None and dt.storage == "pyarrow":
            return dt
    except Exception:
        pass
    return None


def prepare_strings(from_list, to_list):
    """Arrow arrays of the string lists (the only per-string host work of the assembly); callers build them
    while the GPU is still scoring and pass them to assemble_matches(prepared=...)."""
    dt = _str_dtype()
    if dt is None or len(from_list) == 0:
        return None
    from ..strings import ARROW_CACHE

    def arrow_of(lst):
        hit = ARROW_CACHE.get(id(lst))
        if hit is not None and hit[0] is lst:               # packed (and converted) moments ago by the vectoriser
            return hit[1]
        return pa.array(lst, type=pa.large_string())
    same = to_list is None or to_list is from_list
    to_pa = arrow_of(from_list if same else to_list)
    from_pa = to_pa if same else arrow_of(from_list)
    return from_pa, to_pa


def assemble_matches(from_list, to_list, top_idx: np.ndarray, top_val: np.ndarray, prepared=None):
    """top_idx int32[n,k] (global to-index, -1 = none), top_val float64[n,k] (unrounded scores).
    Columns From, To, Similarity, To_2, Similarity_2, ... ; similarities rounded to 3 decimals
    (_utils.py:102); Similarity < 0.001 -> 0.0 and To -> None (_utils.py:119-123)."""
    same = to_list is None or to_list is from_list
    if to_list is None:
        to_list = from_list
    n, k = top_idx.shape
    LAST_TAIL["d2h_bytes"], LAST_TAIL["device"] = int(top_idx.nbytes + top_val.nbytes), False
    # column-major working copies: every per-column array below is contiguous
    sims_t = np.round(np.ascontiguousarray(top_val.T), 3)
    idx_t = np.ascontiguousarray(top_idx.T)
    low_t = sims_t < 0.001
    low_t |= idx_t < 0
    sims_t[low_t] = 0.0
    names = ["To" if r == 0 else f"To_{r + 1}" for r in range(k)]
    snames = ["Similarity" if r == 0 else f"Similarity_{r + 1}" for r in range(k)]
    dt = _str_dtype()
    cols = {}
    if dt is not None and n > 0:
        AT = dt.construct_array_type()
        if prepared is not None:
            from_pa, to_pa = prepared
        else:
            from_pa, to_pa = prepare_strings(from_list, None if same else to_list)
        cols["From"] = pd.Series(AT(from_pa, dtype=dt), copy=False)

        def gather(r):
            ia = pa.array(idx_t[r], mask=low_t[r])            # masked slots become nulls (their index value is ignored)
            return to_pa.take(ia)

        taken = list(_pool().map(gather, range(k))) if (k > 1 and n >= 20000) else [gather(r) for r in range(k)]
        for r in range(k):
            cols[names[r]] = pd.Series(AT(taken[r], dtype=dt), copy=False)
            cols[snames[r]] = sims_t[r]
        return pd.DataFrame(cols, copy=False)
    # generic path (no Arrow-backed str dtype): object columns, explicit dtype so pandas infers nothing
    to_arr = np.empty(len(to_list) + 1, dtype=object)
    to_arr[:-1] = to_list
    to_arr[-1] = None
    cols["From"] = pd.Series(list(from_list), dtype=object)
    for r in range(k):
        idx = np.where(low_t[r], len(to_list), idx_t[r].astype(np.int64))
        cols[names[r]] = pd.Series(to_arr[idx], dtype=object)
        cols[snames[r]] = sims_t[r]
    return pd.DataFrame(cols)


LAST_TAIL = {"d2h_bytes": 0, "device": False}               # bytes of the most recent frame tail's D2H (bench.py reports them)


def device_tail_available(*staged):
    """The frame tail can run on the device (K5) when every list involved is ASCII and pandas has its Arrow-backed str dtype."""
    return _str_dtype() is not None and all(s is not None and getattr(s, "ascii", False) for s in staged)


def arrow_from_staged(S, lo=0, hi=None):
    """Zero-copy Arrow view of an ASCII string list packed by the host (blob bytes + int64 offsets)."""
    n = S.n if hi is None else hi
    arr = pa.LargeStringArray.from_buffers(S.n, pa.py_buffer(S.host_off), pa.py_buffer(S.host_blob))
    return arr if (lo == 0 and n == S.n) else arr.slice(lo, n - lo)


def assemble_matches_device(from_arrow, to_blob, to_off, top_idx, top_val) -> pd.DataFrame:
    """K5: the frame tail of polyfuzz/models/_utils.py:104-125 on the device.  top_idx / top_val are the DEVICE top-k arrays,
    to_blob / to_off the device-resident to-list (int32 code points of an ASCII list, int64 offsets).  Rounding, the
    `< 0.001 -> None` rule and the per-rank string gathers run in two kernels; one D2H brings the finished columns back and
    Arrow / pandas wrap them without copying."""
    import ctypes
    import torch
    from .. import _lib
    from ..engine import _p, _stream, _ws
    n, k = top_idx.shape
    dev = top_idx.device
    dt = _str_dtype()
    AT = dt.construct_array_type()
    nw = (n + 31) // 32
    top_idx = top_idx.contiguous(); top_val = top_val.contiguous()
    sims = torch.empty(k * n, dtype=torch.float64, device=dev)
    pos = torch.empty(k * n + 1, dtype=torch.int64, device=dev)                 # byte positions: a frame may hold >= 2 GiB of strings
    bitmap = torch.empty(k * nw, dtype=torch.int32, device=dev)
    ws_bytes = _lib.load().pfz_frame_tail_ws_bytes(k * n)
    if ws_bytes < 0:
        raise RuntimeError("pfz_frame_tail_ws_bytes failed")
    ws = _ws(ws_bytes)
    _lib.call("pfz_frame_tail_count", _p(top_idx), _p(top_val), n, k, _p(to_off), _p(sims), _p(pos), _p(bitmap), _p(ws), ws.numel(),
              _stream())
    total = int(pos[-1].item())                               # the one host sync of the tail (everything before it is done by then)
    offsets = torch.empty(k * (n + 1), dtype=torch.int64, device=dev)           # large_string offsets: pandas wraps them without a cast
    data = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
    _lib.call("pfz_frame_tail_copy", _p(top_idx), n, k, _p(to_blob), _p(to_off), _p(pos), _p(offsets), _p(data), _stream())
    # one buffer, one D2H: [sims | offsets | bitmap | data]
    parts = [sims.view(torch.uint8), offsets.view(torch.uint8), bitmap.view(torch.uint8), data[:total]]
    sizes = [p.numel() for p in parts]
    # D2H into a pooled pinned buffer (a pageable destination runs at ~4 GB/s and a fresh 35 MB host allocation costs ~8 ms of
    # page faults).  The frame's columns are zero-copy views of that buffer; it returns to the pool when the last view dies.
    import weakref
    from ..engine import _PINNED_OUT as _PINNED
    dev_all = torch.cat(parts)
    nbytes = dev_all.numel()
    stage = _PINNED.take(nbytes)
    stage[:nbytes].copy_(dev_all, non_blocking=True)
    torch.cuda.current_stream().synchronize()
    host = stage[:nbytes].numpy()
    weakref.finalize(host, _PINNED.give, stage, None)
    LAST_TAIL["d2h_bytes"], LAST_TAIL["device"] = int(host.nbytes) + 4, True
    o = np.cumsum([0] + sizes)
    h_sims = host[o[0]:o[1]].view(np.float64).reshape(k, n)
    h_off = host[o[1]:o[2]].view(np.int64).reshape(k, n + 1)
    h_bm = host[o[2]:o[3]].reshape(k, nw * 4)
    h_data = host[o[3]:o[4]]
    col0 = np.concatenate([[0], np.cumsum(h_off[:, n])])                      # byte range of every column in `data`
    cols = {"From": AT(from_arrow, dtype=dt)}
    for r in range(k):
        arr = pa.LargeStringArray.from_buffers(n, pa.py_buffer(h_off[r]), pa.py_buffer(h_data[col0[r]:col0[r + 1]]), pa.py_buffer(h_bm[r]))
        cols["To" if r == 0 else f"To_{r + 1}"] = AT(arr, dtype=dt)
        cols["Similarity" if r == 0 else f"Similarity_{r + 1}"] = h_sims[r]
    return pd.DataFrame(cols, copy=False)
