"""K4 host driver: dense cosine top-k of pre-computed embeddings on the tensor cores (include/pfz.h,
pfz_rows_to_bf16 + pfz_dense_cos_topk).  Inputs are l2-normalised and rounded to bf16 (to_bf16_rows); products
accumulate in fp32 (wgmma register accumulators); the ranking key is (score desc, index asc) on those fp32 values, and a
to-row is eligible iff its score > float32(min_similarity) (and it is not the diagonal of a self-match).
The exact mode (stage_exact + dense_topk_exact) returns the canonical fp64 top-k instead: an fp16 tensor-core filter pass,
fp64 re-scoring of its candidates with a per-row certificate, and a brute-force fp64 pass for the rows not certified."""
import numpy as np
import torch

from . import _lib
from .engine import _dev, _p, _stream, _ws, topk_merge

SM_COUNT = 132                     # H100 SXM


def to_bf16_rows(x, normalize=True):
    """ndarray / tensor [n, d] (float32/float64) -> (device bf16 [n, d_pad], the device input), d_pad = d rounded up to 8
    (at least 8), padding columns +0.  normalize=False: each element is float32(x) rounded to the nearest even bf16.
    normalize=True: each element is a faithful bf16 rounding of x / ||x|| (one of its two bf16 neighbours) wherever that is
    at least 2^-100 in magnitude, and x and 2^e x stage to the same bits at any finite scale; zero rows stay zero."""
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
    if k < 1:
        raise NotImplementedError("dense top_n must be >= 1")
    if k > 32:
        idx, val, _ = dense_topn_bounded(x_bf16, y_bf16, k, min_similarity, self_match, from_index_base, to_index_base, n_splits)
        return idx, val
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


# ---- exact mode (Embeddings(precision="fp64")): the canonical fp64 top-k, bit for bit (DESIGN.md 2 and 4.6) ----------------

class ExactRows:
    """One side staged for the exact mode: canonical l2-normalised fp64 rows `f64` and their fp16 rounding `f16` (both
    [n, d_pad], zero-padded), per-row upper bounds `norm16` >= ||f16 row|| and `err16` >= ||f64 row - f16 row||, and `maxima`
    (float64[2], on the device) = the largest of each."""
    __slots__ = ("f64", "f16", "norm16", "err16", "maxima")

    @property
    def n(self):
        return self.f64.shape[0]

    @property
    def d_pad(self):
        return self.f64.shape[1]


def stage_exact(x):
    """ndarray / tensor [n, d] (float32/float64) -> ExactRows on the device (pfz_rows_prep_exact).  fp32 inputs widen exactly."""
    dev = _dev()
    if isinstance(x, np.ndarray):
        if x.dtype not in (np.float32, np.float64):
            x = x.astype(np.float64)
        t = torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    else:
        t = x.to(dev)
        if t.dtype not in (torch.float32, torch.float64):
            t = t.double()
        t = t.contiguous()
    if t.dim() != 2:
        raise ValueError("embeddings must be a 2-D array [n, d]")
    n, d = t.shape
    d_pad = max(8, (d + 7) // 8 * 8)
    rows = max(n, 1)
    s = ExactRows()
    s.f64 = torch.empty((rows, d_pad), dtype=torch.float64, device=dev)
    s.f16 = torch.empty((rows, d_pad), dtype=torch.float16, device=dev)
    s.norm16 = torch.empty(rows, dtype=torch.float64, device=dev)
    s.err16 = torch.empty(rows, dtype=torch.float64, device=dev)
    s.maxima = torch.empty(2, dtype=torch.float64, device=dev)
    _lib.call("pfz_rows_prep_exact", _p(t), int(t.dtype == torch.float64), int(t.stride(0)) if n else d, n, d, d_pad,
              _p(s.f64), _p(s.f16), _p(s.norm16), _p(s.err16), _p(s.maxima), _stream())
    s.f64, s.f16, s.norm16, s.err16 = s.f64[:n], s.f16[:n], s.norm16[:n], s.err16[:n]
    return s


def k_cand_for(k):
    """Filter candidates per row for a top-k (DESIGN.md 4.6): the largest list of the kernel instantiation (KMAX 10 / 16 / 32)
    that holds about 2k + 4.  The KMAX = 32 instantiation spills registers and filtered C4 5.5x slower than KMAX = 16, so k up
    to 12 takes 16 candidates (C4, k = 10: 0.02 % of the rows then need the fallback)."""
    k = int(k)
    return 10 if k <= 3 else 16 if k <= 12 else 32


def candidates_f16(xs, ys, k_cand, min_similarity=0.0, self_match=False, from_index_base=0, to_index_base=0, n_splits=None):
    """Filter pass of the exact mode (pfz_dense_cos_topk_f16, + pfz_topk_merge over splits): per from-row the k_cand best
    fp32 scores of fp16(x~) . fp16(y~) above min_similarity minus the a-priori margin.  Returns (idx int32, val float64)."""
    dev = _dev()
    n_from, d_pad = xs.f16.shape
    n_to = ys.n
    n_mblocks = (n_from + 127) // 128
    n_ntiles = (n_to + 127) // 128
    if n_splits is None:
        n_splits = max(1, min(n_ntiles, (2 * SM_COUNT + n_mblocks - 1) // n_mblocks))
    n_splits = max(1, min(int(n_splits), n_ntiles))
    ti = torch.empty((n_splits, n_from, k_cand), dtype=torch.int32, device=dev)
    tv = torch.empty((n_splits, n_from, k_cand), dtype=torch.float64, device=dev)
    _lib.call("pfz_dense_cos_topk_f16", _p(xs.f16), _p(ys.f16), n_from, n_to, d_pad, k_cand, float(min_similarity), int(bool(self_match)),
              int(from_index_base), int(to_index_base), n_splits, _p(ti), _p(tv), _stream())
    if n_splits > 1:
        return topk_merge(ti, tv, k_cand)
    return ti[0], tv[0]


def exact_rescore(xs, ys, cand_idx, cand_val, k, min_similarity=0.0, self_match=False, from_index_base=0, to_index_base=0):
    """Canonical fp64 top-k of each row's filter candidates and its certificate (pfz_dense_exact_rescore).
    Returns (idx, val, fb_rows, fb_count): fb_rows[:fb_count] are the rows left to exact_fallback."""
    dev = _dev()
    n_from = xs.n
    idx = torch.empty((n_from, k), dtype=torch.int32, device=dev)
    val = torch.empty((n_from, k), dtype=torch.float64, device=dev)
    fb_rows = torch.empty(max(n_from, 1), dtype=torch.int32, device=dev)
    fb_count = torch.empty(1, dtype=torch.int32, device=dev)
    _lib.call("pfz_dense_exact_rescore", _p(xs.f64), _p(ys.f64), n_from, ys.n, xs.d_pad, k, int(cand_idx.shape[1]), _p(cand_idx.contiguous()),
              _p(cand_val.contiguous()), _p(xs.norm16), _p(xs.err16), _p(ys.maxima), float(min_similarity), int(bool(self_match)),
              int(from_index_base), int(to_index_base), _p(idx), _p(val), _p(fb_rows), _p(fb_count), _stream())
    return idx, val, fb_rows, fb_count


def exact_fallback(xs, ys, idx, val, fb_rows, fb_count, min_similarity=0.0, self_match=False, from_index_base=0, to_index_base=0):
    """Canonical top-k over every to-row for the listed rows, written into idx / val in place (pfz_dense_exact_fallback)."""
    n_from, k = idx.shape
    ws = _ws(_lib.load().pfz_dense_exact_fallback_ws_bytes(n_from, ys.n, k))
    _lib.call("pfz_dense_exact_fallback", _p(xs.f64), _p(ys.f64), n_from, ys.n, xs.d_pad, k, float(min_similarity), int(bool(self_match)),
              int(from_index_base), int(to_index_base), _p(fb_rows), _p(fb_count), _p(idx), _p(val), _p(ws), _stream())


def dense_topk_exact(xs, ys, k, min_similarity=0.0, self_match=False, from_index_base=0, to_index_base=0, n_splits=None, k_cand=None):
    """Canonical fp64 cosine top-k of two ExactRows (stage_exact).  Returns (idx int32[n_from,k] global to-indices or -1,
    val float64[n_from,k], fallback row count int32[1] on the device); no host synchronisation."""
    dev = _dev()
    k = int(k)
    if k < 1:
        raise NotImplementedError("dense top_n must be >= 1")
    if xs.d_pad != ys.d_pad:
        raise ValueError(f"embedding widths differ: {xs.d_pad} vs {ys.d_pad} (padded)")
    if k > 32:
        idx, val, n_over = dense_topn_bounded(xs, ys, k, min_similarity, self_match, from_index_base, to_index_base, n_splits)
        return idx, val, torch.full((1,), n_over, dtype=torch.int32, device=dev)
    if xs.n == 0:
        return (torch.empty((0, k), dtype=torch.int32, device=dev), torch.empty((0, k), dtype=torch.float64, device=dev),
                torch.zeros(1, dtype=torch.int32, device=dev))
    kc = max(k, min(32, int(k_cand) if k_cand else k_cand_for(k)))
    ci, cv = candidates_f16(xs, ys, kc, min_similarity, self_match, from_index_base, to_index_base, n_splits)
    idx, val, fb_rows, fb_count = exact_rescore(xs, ys, ci, cv, k, min_similarity, self_match, from_index_base, to_index_base)
    exact_fallback(xs, ys, idx, val, fb_rows, fb_count, min_similarity, self_match, from_index_base, to_index_base)
    return idx, val, fb_count


# ---- top_n > 32, both precisions (DESIGN.md 4.7): bound, threshold pass, select -----------------------------------------------

TOPN_WS_BYTES = 512 << 20          # bound lists + candidate buffers of one chunk of from-rows
TOPN_LIST = 16                     # the bound pass runs the KMAX = 16 instantiation


def topn_cap_for(k):
    """Default candidate slots per row of the threshold pass: 4k rounded up to 32, at least 256."""
    return max(256, (4 * int(k) + 31) // 32 * 32)


def _splits(rows, n_ntiles):
    mb = (rows + 127) // 128
    return max(1, min(n_ntiles, (2 * SM_COUNT + mb - 1) // mb))


def dense_topn_bounded(x, y, k, min_similarity=0.0, self_match=False, from_index_base=0, to_index_base=0, n_splits=None,
                       cap=None, chunk_rows=None, events=None):
    """Top-k of any size k (DESIGN.md 4.7); dense_topk and dense_topk_exact take this path for k > 32, and for k <= 32 it returns
    what they return.  x, y: bf16 rows (to_bf16_rows) or ExactRows (stage_exact: the exact mode).

    Per chunk of from-rows: a bound pass (the top-16 kernel with >= 2k/16 unmerged splits, then pfz_dense_topn_bound), the
    threshold pass (pfz_dense_cos_cand[_f16], `cap` slots per row), in the exact mode the canonical re-score, and the select.
    Rows with more than `cap` candidates are then re-run with the exact capacity; that takes one device-to-host read (their
    number and the largest count).  Returns (idx int32[n_from,k], val float64[n_from,k], overflow row count).
    `events` (a list) receives (stage name, CUDA event) pairs at the stage boundaries."""
    dev = _dev()
    k = int(k)
    if k < 1:
        raise NotImplementedError("dense top_n must be >= 1")
    exact = isinstance(x, ExactRows)
    xop, yop = (x.f16, y.f16) if exact else (x, y)
    n_from, d = xop.shape
    n_to = yop.shape[0]
    idx = torch.empty((n_from, k), dtype=torch.int32, device=dev)
    val = torch.empty((n_from, k), dtype=torch.float64, device=dev)
    if n_from == 0:
        return idx, val, 0
    thr = float(min_similarity)
    sel_thr = thr if exact else float(np.float32(thr))   # the bf16 kernel compares fp32 scores with float(min_similarity)
    st = _stream()
    n_ntiles = (n_to + 127) // 128
    s_min = -(-2 * k // TOPN_LIST)
    cap = max(1, min(n_to, int(cap) if cap else topn_cap_for(k)))
    if chunk_rows is None:
        per_row = 12 * (min(n_ntiles, max(s_min, 4)) * TOPN_LIST + cap) + 16
        chunk_rows = max(128, TOPN_WS_BYTES // per_row // 128 * 128)
    chunk_rows = max(1, int(chunk_rows))
    topk_fn = "pfz_dense_cos_topk_f16" if exact else "pfz_dense_cos_topk"
    cand_fn = "pfz_dense_cos_cand_f16" if exact else "pfz_dense_cos_cand"

    def mark(name):
        if events is not None:
            e = torch.cuda.Event(enable_timing=True); e.record(); events.append((name, e))

    def run_rows(xg, row_map, out_lo, thr_rows, cnt_rows, c, timed=True):
        """Threshold pass, exact re-score and select of the rows xg (output rows row_map, or out_lo + r)."""
        m = xg.shape[0]
        ci = torch.empty((m, c), dtype=torch.int32, device=dev)
        cv = torch.empty((m, c), dtype=torch.float64, device=dev)
        sp = max(1, min(n_ntiles, int(n_splits) if n_splits else _splits(m, n_ntiles)))
        _lib.call(cand_fn, _p(xg), _p(yop), m, n_to, d, thr, _p(thr_rows), int(to_index_base), sp, c, _p(ci), _p(cv), _p(cnt_rows), st)
        if timed:
            mark("select")
        if exact:
            xf = x.f64 if row_map is not None else x.f64[out_lo:out_lo + m]
            _lib.call("pfz_dense_topn_exact_rescore", _p(xf), _p(y.f64), m, d, _p(row_map), int(to_index_base), c, _p(ci), _p(cv),
                      _p(cnt_rows), st)
        oi = idx if row_map is not None else idx[out_lo:out_lo + m]
        ov = val if row_map is not None else val[out_lo:out_lo + m]
        fb = int(from_index_base) + (0 if row_map is not None else out_lo)
        _lib.call("pfz_dense_topn_select", _p(ci), _p(cv), _p(cnt_rows), m, c, k, sel_thr, int(bool(self_match)), fb, _p(row_map),
                  _p(oi), _p(ov), st)

    row_thr = torch.empty(n_from, dtype=torch.float32, device=dev)
    counts = torch.empty(n_from, dtype=torch.int32, device=dev)
    for lo in range(0, n_from, chunk_rows):
        hi = min(n_from, lo + chunk_rows)
        rows = hi - lo
        mark("bound")
        s = max(1, min(n_ntiles, max(s_min, int(n_splits) if n_splits else _splits(rows, n_ntiles))))
        li = torch.empty((s, rows, TOPN_LIST), dtype=torch.int32, device=dev)
        lv = torch.empty((s, rows, TOPN_LIST), dtype=torch.float64, device=dev)
        _lib.call(topk_fn, _p(xop[lo:hi]), _p(yop), rows, n_to, d, TOPN_LIST, thr, int(bool(self_match)), int(from_index_base) + lo,
                  int(to_index_base), s, _p(li), _p(lv), st)
        _lib.call("pfz_dense_topn_bound", _p(li), _p(lv), s, rows, TOPN_LIST, k, int(exact),
                  _p(x.norm16[lo:hi] if exact else None), _p(x.err16[lo:hi] if exact else None), _p(y.maxima if exact else None), d,
                  thr, _p(row_thr[lo:hi]), st)
        del li, lv
        mark("threshold")
        run_rows(xop[lo:hi], None, lo, row_thr[lo:hi], counts[lo:hi], cap)
    mark("overflow")
    over = counts > cap
    n_over, max_cnt = torch.stack([over.sum(), counts.max().long()]).tolist()   # the one device-to-host read
    if n_over:
        rows_over = torch.argsort(over.int(), descending=True, stable=True)[:n_over].int()
        chunk2 = max(1, TOPN_WS_BYTES // (12 * max_cnt))
        for a in range(0, n_over, chunk2):
            r = rows_over[a:a + chunk2]
            cnt2 = torch.empty(len(r), dtype=torch.int32, device=dev)
            run_rows(xop.index_select(0, r), r, 0, row_thr.index_select(0, r), cnt2, max_cnt, timed=False)
    mark("end")
    return idx, val, int(n_over)
