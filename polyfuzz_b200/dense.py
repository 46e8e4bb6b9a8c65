"""K4 host driver: dense cosine top-k of pre-computed embeddings on the tensor cores (include/pfz.h,
pfz_rows_to_bf16 + pfz_dense_cos_topk).  Inputs are rounded to bf16 (after l2 normalisation in fp32);
products accumulate in fp32 (wgmma register accumulators); the ranking key is (score desc, index asc) on those fp32 values."""
import numpy as np
import torch

from . import _lib
from .engine import _dev, _p, _stream, topk_merge

SM_COUNT = 132                     # H100 SXM


def to_bf16_rows(x, normalize=True):
    """ndarray / tensor [n, d] (float32/float64) -> device bf16 [n, d_pad] (d_pad = d rounded up to 8)."""
    dev = _dev()
    if isinstance(x, np.ndarray):
        if x.dtype not in (np.float32, np.float64):
            x = x.astype(np.float32)
        t = torch.from_numpy(np.ascontiguousarray(x)).to(dev, non_blocking=False)
    else:
        t = x.to(dev)
        if t.dtype not in (torch.float32, torch.float64):
            t = t.float()
        t = t.contiguous()
    if t.dim() != 2:
        raise ValueError("embeddings must be a 2-D array [n, d]")
    n, d = t.shape
    d_pad = max(8, (d + 7) // 8 * 8)
    out = torch.empty((max(n, 1), d_pad), dtype=torch.bfloat16, device=dev)
    _lib.call("pfz_rows_to_bf16", _p(t), int(t.dtype == torch.float64), int(t.stride(0)) if n else d, n, d, d_pad, int(bool(normalize)),
              _p(out), _stream())
    return out[:n], t


def dense_topk(x_bf16, y_bf16, k, min_similarity=0.0, self_match=False, from_index_base=0, to_index_base=0, n_splits=None):
    """top-k of X * Y^T.  Returns (idx int32[n_from,k] global to-indices or -1, val float64[n_from,k])."""
    dev = _dev()
    n_from, d = x_bf16.shape
    n_to = y_bf16.shape[0]
    k = int(k)
    if not 1 <= k <= 32:
        raise NotImplementedError("dense top_n is limited to 32 per call")
    if n_from == 0:
        return torch.empty((0, k), dtype=torch.int32, device=dev), torch.empty((0, k), dtype=torch.float64, device=dev)
    n_mblocks = (n_from + 127) // 128
    n_ntiles = (n_to + 127) // 128                     # 128-wide to-tiles (pfz_dense.cu DN)
    if n_splits is None:
        n_splits = max(1, min(n_ntiles, (2 * SM_COUNT + n_mblocks - 1) // n_mblocks))
    n_splits = max(1, min(int(n_splits), n_ntiles))
    ti = torch.empty((n_splits, n_from, k), dtype=torch.int32, device=dev)
    tv = torch.empty((n_splits, n_from, k), dtype=torch.float64, device=dev)
    _lib.call("pfz_dense_cos_topk", _p(x_bf16), _p(y_bf16), n_from, n_to, d, k, float(min_similarity), int(bool(self_match)),
              int(from_index_base), int(to_index_base), n_splits, _p(ti), _p(tv), _stream())
    if n_splits > 1:
        return topk_merge(ti, tv, k)
    return ti[0], tv[0]
