"""Device-side engine: thin Python drivers over the C ABI (include/pfz.h).  PyTorch is used only for
device memory, streams and (in distributed.py) NCCL -- every kernel is in libpfz.so.

Classes
    NgramTfidf   K1: fit / transform of the char-n-gram TF-IDF vectoriser -> CSR tensors in HBM
    SparseIndex  inverted index of a to-matrix (term x to-tile posting segments)
Functions
    index_for    the K2 index of a TF-IDF to-matrix: picks the variant, and replaces it when from-rows outgrow its kernel
    spcos_topk   K2: fused sparse cosine + per-row top-k (pages of 32 for larger k), tile splits + merge
The TF-IDF path K1 -> index -> K2 is driven by distributed.tfidf_topk_sharded, on one GPU and on many.
"""
import ctypes
import os

import numpy as np
import torch

from . import _lib
from .strings import pack_utf32, pack_strings, ngram_slot_bounds

FLAG_CLEAN, FLAG_REMOVE_SPACE = 1, 2
WARP_ROW_SLOTS, MAX_ROW_SLOTS = 256, 8192
DENSE_CODE_SPACE_MAX = 1 << 24
CLEAN_BASE = 38
N_CODE_POINTS = 0x110000


def _dev():
    if not torch.cuda.is_available():
        raise RuntimeError("polyfuzz_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


class _PinnedPool:
    """Reusable pinned staging buffers (cudaHostAlloc per call costs more than the copy for MB-sized
    inputs).  A buffer is handed out again only after the H2D copy that used it has completed."""

    def __init__(self):
        self.free = []          # [(tensor uint8, event or None)]

    def take(self, nbytes):
        best = None
        for i, (buf, ev) in enumerate(self.free):
            if buf.numel() >= nbytes and (best is None or buf.numel() < self.free[best][0].numel()):
                best = i
        if best is not None:
            buf, ev = self.free.pop(best)
            if ev is not None:
                ev.synchronize()
            return buf
        size = max(1 << 16, 1 << int(nbytes - 1).bit_length())
        return torch.empty(size, dtype=torch.uint8).pin_memory()

    def give(self, buf, ev):
        if len(self.free) < 16:
            self.free.append((buf, ev))


_PINNED = _PinnedPool()          # H2D staging
_PINNED_OUT = _PinnedPool()      # result buffers of the frame tail (kept apart: a small H2D must never grab a 64 MB result buffer)


def _to_dev(arr, dtype=None):
    """numpy -> device tensor via pooled pinned staging (async H2D on the current stream)."""
    dev = _dev()                                           # fail loudly without a GPU, before any work
    arr = np.ascontiguousarray(arr)
    t = torch.from_numpy(arr)
    if dtype is not None:
        t = t.view(dtype)
    if t.numel() == 0:
        return torch.empty(0, dtype=t.dtype, device=dev)
    nbytes = arr.nbytes
    stage = _PINNED.take(nbytes)
    stage[:nbytes].copy_(torch.from_numpy(arr.reshape(-1).view(np.uint8)))
    out = torch.empty(t.shape, dtype=t.dtype, device=dev)
    out.view(torch.uint8).reshape(-1).copy_(stage[:nbytes], non_blocking=True)
    ev = torch.cuda.Event(); ev.record()
    _PINNED.give(stage, ev)
    return out


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=_dev())


class CsrMatrix:
    """l2-normalised TF-IDF rows in HBM: int32 indptr[n+1], int32 indices[cap], float64 data[cap]
    (cap >= nnz; nnz = indptr[n])."""

    def __init__(self, indptr, indices, data, n_rows, n_cols):
        self.indptr, self.indices, self.data = indptr, indices, data
        self.n_rows, self.n_cols = n_rows, n_cols

    def to_scipy(self):
        import scipy.sparse as sp
        ip = self.indptr.cpu().numpy()
        nnz = int(ip[-1]) if len(ip) else 0
        return sp.csr_matrix((self.data[:nnz].cpu().numpy(), self.indices[:nnz].cpu().numpy(), ip),
                             shape=(self.n_rows, self.n_cols))

    @staticmethod
    def from_scipy(m):
        m = m.tocsr(); m.sort_indices()
        return CsrMatrix(_to_dev(m.indptr.astype(np.int32)), _to_dev(m.indices.astype(np.int32)),
                         _to_dev(m.data.astype(np.float64)), m.shape[0], m.shape[1])


class StagedStrings:
    """One string list packed and resident in HBM (UTF-32 blob, offsets, n-gram slot prefix)."""
    __slots__ = ("n", "n_chars", "d_blob", "d_off", "occ_ptr", "d_long", "n_long", "cap", "h2d_bytes", "lo", "hi", "max_slots",
                 "ascii", "host_blob", "host_off")


def stage_strings(strings, lo, hi):
    """Host marshalling + H2D of one list (the only per-string Python work on the path)."""
    blob, offsets, _arrow = pack_strings(strings)
    slots, occ = ngram_slot_bounds(offsets, lo, hi)
    if len(slots) and slots.max() > MAX_ROW_SLOTS:
        r = int(slots.argmax())
        raise ValueError(f"string {r} has {int(slots[r])} n-gram slots; the vectoriser supports at most "
                         f"{MAX_ROW_SLOTS} per string")
    long_rows = np.nonzero(slots > WARP_ROW_SLOTS)[0].astype(np.int32)
    S = StagedStrings()
    S.n, S.n_chars, S.cap, S.lo, S.hi = len(strings), int(blob.size), int(occ[-1]), lo, hi
    S.max_slots = int(slots.max()) if len(slots) else 0        # upper bound of any row's nnz
    S.ascii = blob.dtype == np.uint8                           # bytes == code points: the frame tail can run on the device (K5)
    S.host_blob, S.host_off = (blob, offsets) if S.ascii else (None, None)
    if blob.size == 0:
        S.d_blob = torch.zeros(1, dtype=torch.int32, device=_dev())
    elif blob.dtype == np.uint8:                              # ASCII list: 1 byte per code point over PCIe, widened in HBM
        S.d_blob = _to_dev(blob).to(torch.int32)
    else:
        S.d_blob = _to_dev(blob.view(np.int32), torch.int32)
    S.d_off = _to_dev(offsets)
    S.occ_ptr = _to_dev(occ)
    S.n_long = len(long_rows)
    S.d_long = _to_dev(long_rows) if S.n_long else None
    S.h2d_bytes = blob.nbytes + offsets.nbytes + occ.nbytes + long_rows.nbytes
    return S


_IDF_TABLES = {}


def _idf_table(n_docs):
    """Device table idf(df) for df = 0..n_docs with scikit-learn's expression evaluated by numpy on the host (cached per n_docs)."""
    key = (int(n_docs), torch.cuda.current_device())
    t = _IDF_TABLES.get(key)
    if t is None:
        tab = np.log((n_docs + 1.0) / (np.arange(0, n_docs + 1, dtype=np.float64) + 1.0)) + 1.0
        if len(_IDF_TABLES) > 8:
            _IDF_TABLES.clear()
        t = _IDF_TABLES[key] = _to_dev(tab)
    return t


class _Rows:
    """Stage-A result for one string list: per-row sorted distinct n-gram codes + counts."""
    __slots__ = ("n", "occ_ptr", "codes", "tf", "row_cnt", "cap", "_keep")


def _pow2(n):
    return 1 << max(int(n - 1).bit_length(), 1)


def _sorted_unique(keys, n_keys, cap, d_nv):
    """Sort `keys` (uint64 codes carried in int64, power-of-two length, ~0 after the first *n_keys) and run-length them:
    -> (distinct codes int64[cap] ascending, multiplicities int32[cap]); *d_nv (device int32[1]) = how many."""
    n = keys.numel()
    _lib.call("pfz_sort_u64", _p(keys), n, _stream())
    d_vocab = torch.empty(cap, dtype=torch.int64, device=keys.device)
    d_cnt = torch.empty(cap, dtype=torch.int32, device=keys.device)
    ws = _ws(n * 8 + 256 + _lib.load().pfz_scan_ws_bytes(n))
    _lib.call("pfz_vocab_from_sorted", _p(keys), n, _p(n_keys), _p(d_vocab), _p(d_cnt), _p(d_nv), _p(ws), _stream())
    return d_vocab, d_cnt


def _vocab_of_rows(rows, d_nv):
    """Vocabulary of stage-A rows for a large code space (gather + bitonic sort + run-length): (codes, df); *d_nv = V."""
    total = sum(r.cap for r in rows)
    keys = torch.full((_pow2(total),), -1, dtype=torch.int64, device=_dev())       # ~0 padding
    cursor = torch.zeros(1, dtype=torch.int64, device=_dev())
    for r in rows:
        _lib.call("pfz_gather_codes", _p(r.codes), _p(r.occ_ptr), _p(r.row_cnt), r.n, _p(keys), _p(cursor), _stream())
    return _sorted_unique(keys, cursor, max(total, 1), d_nv)


def _vocab_across_ranks(rows, comm, d_nv):
    """Multi-GPU fit with a code space too large for a dense df table.  The global vocabulary is the sorted union of the ranks'
    local vocabularies (one variable-length all-gather, then the same sort on every rank); the global df is each rank's local
    df stored at its codes' global ranks and summed over the ranks (one integer all-reduce).  Every rank derives the same bits
    as a single-GPU fit of the whole corpus, and every rank raises its empty-vocabulary ValueError, after the exchange."""
    dev = _dev()
    loc_nv = torch.zeros(1, dtype=torch.int32, device=dev)
    loc_vocab, loc_df = _vocab_of_rows(rows, loc_nv)
    gathered, lengths = comm.all_gather_varlen(loc_vocab, loc_nv)              # int64[G, max V_r], ~0 padding
    n_keys = sum(lengths)
    keys = torch.full((_pow2(gathered.numel()),), -1, dtype=torch.int64, device=dev)
    keys[:gathered.numel()] = gathered.reshape(-1)
    # (the multiplicities of the union count ranks, not documents: unused)
    d_vocab, _ = _sorted_unique(keys, torch.tensor([n_keys], dtype=torch.int64, device=dev), max(n_keys, 1), d_nv)
    V = int(d_nv.item())
    if V == 0:
        raise ValueError("empty vocabulary; perhaps the documents only contain stop words")
    d_df = torch.zeros(V, dtype=torch.int32, device=dev)
    _lib.call("pfz_df_scatter", _p(loc_vocab), _p(loc_df), _p(loc_nv), int(loc_vocab.numel()), _p(d_vocab), V, _p(d_df), _stream())
    comm.all_reduce_sum(d_df)
    return d_vocab, d_df


class NgramTfidf:
    """GPU statement of `TfidfVectorizer(min_df=1, analyzer=TFIDF._create_ngrams)` as the reference
    uses it (polyfuzz/models/_tfidf.py:102-118).  fit() learns vocabulary (alphabetical == ascending
    n-gram code) and idf; transform() emits the l2-normalised CSR in HBM."""

    def __init__(self, n_gram_range=(3, 3), clean_string=True, remove_space_ngrams=True):
        lo, hi = int(n_gram_range[0]), int(n_gram_range[1])
        if not (1 <= lo <= hi <= 8):
            raise ValueError(f"n_gram_range {n_gram_range} unsupported (1 <= lo <= hi <= 8)")
        self.lo, self.hi = lo, hi
        self.clean = bool(clean_string)
        self.remove_space = bool(remove_space_ngrams)
        self.flags = (FLAG_CLEAN if self.clean else 0) | (FLAG_REMOVE_SPACE if self.remove_space else 0)
        self.base = CLEAN_BASE if self.clean else None
        self.alphabet = None            # raw mode: sorted code points of the fit corpus (numpy uint32)
        self._h_vocab_keys = None       # numpy uint64[V] ascending (host copies are made lazily: pickling / inspection)
        self._h_idf = None              # numpy float64[V]
        self._h_df = None
        self._n_vocab = 0
        self._sum_df_sq = None          # sum_t df_t^2 (density of the fitted corpus), from the fit's one small D2H
        self.n_fit_docs = 0
        self.max_row_nnz = 0            # upper bound over every list seen (fit and transform)
        self._d_sym = self._d_vocab = self._d_idf = self._d_rank = self._d_df = None

    # ---- pickling: device tensors are rebuilt lazily ---------------------------------------------
    def __getstate__(self):
        if self._n_vocab:
            self.vocab_keys, self.df, self.idf                  # materialise the host copies
        st = dict(self.__dict__)
        for k in ("_d_sym", "_d_vocab", "_d_idf", "_d_rank", "_d_df"):
            st[k] = None
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)
        self.__dict__.setdefault("_d_df", None)

    @property
    def n_vocab(self):
        return self._n_vocab

    # host copies of the fitted state, fetched from the device on first use
    @property
    def vocab_keys(self):
        if self._h_vocab_keys is None and self._n_vocab and self._d_vocab is not None:
            self._h_vocab_keys = self._d_vocab[:self._n_vocab].cpu().numpy().view(np.uint64)
        return self._h_vocab_keys

    @property
    def df(self):
        if self._h_df is None and self._n_vocab and self._d_df is not None:
            self._h_df = self._d_df[:self._n_vocab].cpu().numpy().astype(np.int64)
        return self._h_df

    @property
    def idf(self):
        if self._h_idf is None and self._n_vocab and self._d_idf is not None:
            self._h_idf = self._d_idf[:self._n_vocab].cpu().numpy()
        return self._h_idf

    def code_space(self):
        return int(self.base) ** self.hi

    def vocabulary(self):
        """n-gram strings in column order (decoded from the codes) -- sklearn's sorted vocabulary_."""
        out = []
        if self.clean:
            symbols = [None, " "] + [chr(c) for c in range(48, 58)] + [chr(c) for c in range(97, 123)]
        else:
            symbols = [None] + [chr(int(c)) for c in self.alphabet]
        for key in self.vocab_keys.tolist():
            digs = []
            for _ in range(self.hi):
                digs.append(key % self.base); key //= self.base
            out.append("".join(symbols[d] for d in reversed(digs) if d))
        return out

    def stage(self, strings):
        return stage_strings(strings, self.lo, self.hi)

    # ---- stage A ----------------------------------------------------------------------------------
    def _stage_a(self, S, d_sym, fit=False):
        R = _Rows()
        R.n, R.cap, R.occ_ptr = S.n, S.cap, S.occ_ptr
        R.codes = torch.empty(max(R.cap, 1), dtype=torch.int64, device=_dev())
        R.tf = torch.empty(max(R.cap, 1), dtype=torch.int32, device=_dev())
        R.row_cnt = torch.zeros(max(R.n, 1), dtype=torch.int32, device=_dev())
        _lib.call("pfz_ngram_rows", _p(S.d_blob), _p(S.d_off), R.n, self.lo, self.hi, self.flags, _p(d_sym),
                  int(self.base), _p(R.occ_ptr), _p(S.d_long), S.n_long, _p(R.codes), _p(R.tf), _p(R.row_cnt),
                  _stream())
        R._keep = S
        # upper bound of any row's nnz: the host-side slot bound, tightened to the true maximum (one small D2H) only when
        # the bound alone would rule out the fp32-filter kernels
        if not fit:                                           # (fit folds the true maximum into its one D2H)
            bound = S.max_slots
            if bound > DENSE32_MAX_ROW_NNZ and R.n:
                bound = int(R.row_cnt[:R.n].max().item())
            self.max_row_nnz = max(self.max_row_nnz, bound)
        return R

    def _fit_alphabet(self, staged, comm=None):
        present = torch.zeros(N_CODE_POINTS, dtype=torch.uint8, device=_dev())
        for S in staged:
            if S.n_chars:
                _lib.call("pfz_alphabet_mark", _p(S.d_blob), S.n_chars, _p(present), _stream())
        if comm is not None:
            comm.all_reduce_max(present)
        self.alphabet = np.nonzero(present.cpu().numpy())[0].astype(np.uint32)
        self.base = len(self.alphabet) + 1

    def _sym_table(self):
        if self.clean:
            return None
        if self._d_sym is None:
            tab = np.full(N_CODE_POINTS, 0xFFFFFFFF, dtype=np.uint32)
            tab[self.alphabet] = np.arange(1, len(self.alphabet) + 1, dtype=np.uint32)
            self._d_sym = _to_dev(tab.view(np.int32), torch.int32)
        return self._d_sym

    # ---- fit ----------------------------------------------------------------------------------------
    def fit_rows(self, lists):
        """lists: the fit corpus as 1 or 2 string lists (the reference fits on to_list + from_list,
        _tfidf.py:109).  Returns the stage-A rows of each list so transform need not redo them."""
        return self.fit_staged([self.stage(l) for l in lists])

    def fit_staged(self, staged, counted=None, comm=None, n_docs_total=None):
        """Fit on device-resident lists.  `counted[i]` says whether list i contributes to the vocabulary, df and
        n_docs (on THIS rank): a list that is only scored, such as a from-block of a self-match, is not counted, and a
        list replicated on every rank is counted on rank 0 only.  Multi-GPU (comm given): the
        dense df table and the document count are summed across ranks (one all-reduce), after which
        every rank derives the identical vocabulary and idf.  A code space above DENSE_CODE_SPACE_MAX
        all-gathers the ranks' local vocabularies instead (_vocab_across_ranks)."""
        if counted is None:
            counted = [True] * len(staged)
        if not self.clean:
            self._d_sym = None
            self._fit_alphabet(staged, comm)
        if self.code_space() >= 2 ** 64:
            raise ValueError(f"alphabet of {self.base - 1} symbols with {self.hi}-grams exceeds 64-bit n-gram codes")
        d_sym = self._sym_table()
        rows = [self._stage_a(S, d_sym, fit=True) for S in staged]
        counted_rows = [r for r, c in zip(rows, counted) if c]
        n_docs = sum(r.n for r in counted_rows)
        dev = _dev()
        d_nv = torch.zeros(1, dtype=torch.int32, device=dev)
        cs = self.code_space()
        total_cap = sum(r.cap for r in rows)
        if comm is not None:
            if n_docs_total is not None:
                # the caller knows the global document count (every rank sees the list lengths): no collective, no host sync here;
                # the dense vocabulary buffers are then sized by the code space instead of the summed n-gram slots (the large
                # code space path sizes its buffers from the gathered vocabulary lengths)
                n_docs, total_cap_all = int(n_docs_total), cs
            else:
                meta = torch.tensor([n_docs, total_cap], dtype=torch.int64, device=dev)
                comm.all_reduce_sum(meta)
                n_docs, total_cap_all = int(meta[0].item()), int(meta[1].item())
        else:
            total_cap_all = total_cap
        if total_cap_all == 0:
            raise ValueError("empty vocabulary; perhaps the documents only contain stop words")
        if cs <= DENSE_CODE_SPACE_MAX:
            df_dense = torch.zeros(cs, dtype=torch.int32, device=dev)
            for r in counted_rows:
                _lib.call("pfz_df_dense", _p(r.codes), _p(r.occ_ptr), _p(r.row_cnt), r.n, _p(df_dense), _stream())
            if comm is not None:
                comm.all_reduce_sum(df_dense)
            vmax = min(cs, total_cap_all)
            d_vocab = torch.empty(vmax, dtype=torch.int64, device=dev)
            d_df = torch.empty(vmax, dtype=torch.int32, device=dev)
            d_rank = torch.empty(cs, dtype=torch.int32, device=dev)
            ws = _ws(_lib.load().pfz_scan_ws_bytes(cs))
            _lib.call("pfz_vocab_compact_dense", _p(df_dense), cs, _p(d_vocab), _p(d_df), _p(d_rank), _p(d_nv), _p(ws), _stream())
        elif comm is not None:
            d_vocab, d_df = _vocab_across_ranks(counted_rows, comm, d_nv)
            d_rank = None
        else:
            d_vocab, d_df = _vocab_of_rows(counted_rows, d_nv)
            d_rank = None
        # idf exactly as scikit-learn computes it on the host (sk:feature_extraction/text.py:1679-1694):
        # np.log((n_samples + 1) / (df + 1)) + 1 -- same numpy, same bits as the reference on this machine -- as a TABLE over
        # every possible df (0..n_docs), looked up on the device: no df D2H, no idf H2D, nothing waits for the host.
        d_tab = _idf_table(n_docs)
        d_idf = torch.empty(d_df.numel(), dtype=torch.float64, device=dev)
        _lib.call("pfz_idf_lookup", _p(d_df), _p(d_nv), int(d_df.numel()), _p(d_tab), int(d_tab.numel()), _p(d_idf), _stream())
        # the one small D2H (and host sync) of fit: V, sum df^2 (chooses the K2 variant), the longest row
        dfv = d_df.double()
        vmask = torch.arange(d_df.numel(), device=dev) < d_nv
        mx = torch.stack([r.row_cnt[:r.n].max() if r.n else torch.zeros((), dtype=torch.int32, device=dev) for r in rows]).max()
        stats = torch.stack([d_nv[0].double(), torch.where(vmask, dfv * dfv, torch.zeros_like(dfv)).sum(), mx.double()]).cpu().numpy()
        V = int(stats[0])
        if V == 0:
            raise ValueError("empty vocabulary; perhaps the documents only contain stop words")
        self._n_vocab = V
        self._sum_df_sq = float(stats[1])
        self.max_row_nnz = max(self.max_row_nnz, int(stats[2]))
        self._h_vocab_keys = self._h_df = self._h_idf = None
        self.n_fit_docs = n_docs
        self._d_vocab = d_vocab[:V]
        self._d_df = d_df[:V]
        self._d_rank = d_rank
        self._d_idf = d_idf[:V]
        return rows

    def _ensure_device_state(self):
        if not self._n_vocab:
            raise ValueError("vectoriser is not fitted")
        if self._d_vocab is None:                             # restored from a pickle
            self._d_vocab = _to_dev(self._h_vocab_keys.view(np.int64))
            self._d_idf = _to_dev(self._h_idf)
            self._d_df = _to_dev(self._h_df.astype(np.int32))
            self._d_rank = None
            cs = self.code_space()
            if cs <= DENSE_CODE_SPACE_MAX:
                rank = np.full(cs, -1, dtype=np.int32)
                rank[self.vocab_keys.astype(np.int64)] = np.arange(len(self.vocab_keys), dtype=np.int32)
                self._d_rank = _to_dev(rank)

    # ---- transform ----------------------------------------------------------------------------------
    def rows(self, strings):
        self._ensure_device_state()
        return self._stage_a(strings if isinstance(strings, StagedStrings) else self.stage(strings), self._sym_table())

    def emit(self, R):
        self._ensure_device_state()
        dev = _dev()
        indptr = torch.empty(R.n + 1, dtype=torch.int32, device=dev)
        indices = torch.empty(max(R.cap, 1), dtype=torch.int32, device=dev)
        data = torch.empty(max(R.cap, 1), dtype=torch.float64, device=dev)
        ws = _ws(_lib.load().pfz_scan_ws_bytes(R.n + 1))
        _lib.call("pfz_tfidf_emit", _p(R.codes), _p(R.tf), _p(R.occ_ptr), _p(R.row_cnt), R.n, _p(self._d_rank),
                  _p(self._d_vocab), self.n_vocab, _p(self._d_idf), _p(indptr), _p(indices), _p(data), _p(ws), _stream())
        return CsrMatrix(indptr, indices, data, R.n, self.n_vocab)

    def density(self):
        """Postings visited per scored pair, estimated from the fitted document frequencies:
        sum_t df_t^2 / n_docs^2 (exact for a self-match).  Chooses the K2 variant."""
        if not self.n_fit_docs or not self._n_vocab:
            return None
        if self._sum_df_sq is None:
            d = self.df.astype(np.float64)
            self._sum_df_sq = float((d * d).sum())
        return self._sum_df_sq / float(self.n_fit_docs) ** 2

    def fit(self, strings):
        self.fit_rows([strings])
        return self

    def transform(self, strings):
        return self.emit(self.rows(strings))


# to-tile rows per K2 variant: the list kernel wants many small per-warp arenas (occupancy), the dense
# kernel few large ones (long segments; it pipelines its own loads)
DEFAULT_TILE = {"list": int(os.environ.get("PFZ_TILE_LIST", "512")), "dense": int(os.environ.get("PFZ_TILE_DENSE", "1024")),
                "dense32": int(os.environ.get("PFZ_TILE_DENSE32", "1024")), "block": int(os.environ.get("PFZ_TILE_BLOCK", "4096")),
                "hash": 65536}
# block kernel: the tile above is for 16-bit accumulators; 32-bit ones take half of it, the same accumulator bytes (a 4 096-row
# tile of 32-bit accumulators would not fit a 16-row CTA in shared memory)
BLOCK_TILE_STEP, BLOCK_TILE_MAX = 128, 4096
BLOCK_ROWS = int(os.environ.get("PFZ_BLOCK_ROWS", "8"))           # from-rows (= warps) per CTA of the block kernel: 4, 8 or 16
BLOCK_ACC_BITS = int(os.environ.get("PFZ_BLOCK_ACC_BITS", "16"))  # 16: two accumulators per word (unit 2^-15); 32: one per word (2^-26)


class SparseIndex:
    """Inverted index of a to-matrix shard: postings grouped by (term, to-tile)."""

    def __init__(self, csr: CsrMatrix, tile=None, variant="list"):
        n = csr.n_rows
        self.variant = variant
        if tile is None:
            tile = DEFAULT_TILE[variant]
            if variant == "block" and BLOCK_ACC_BITS != 16:
                tile //= 2
        tile = max(64, min(int(tile), ((max(n, 1) + 63) // 64) * 64))
        self.acc_bits = 32
        if variant == "block":                                # the block kernel scans its accumulators 128 words per warp step
            self.acc_bits = 16 if BLOCK_ACC_BITS == 16 else 32
            step = BLOCK_TILE_STEP * (2 if self.acc_bits == 16 else 1)
            tile = min(BLOCK_TILE_MAX, max(step, (tile + step - 1) // step * step))
        self.tile = tile
        self.n_to = n
        self.n_vocab = csr.n_cols
        self.n_tiles = max(1, (n + tile - 1) // tile)
        ncell = self.n_vocab * self.n_tiles
        dev = _dev()
        self.seg = torch.empty(ncell + 1, dtype=torch.int32, device=dev)
        cap = max(csr.indices.numel(), 1)
        self.post_idx = torch.empty(cap, dtype=torch.int16, device=dev)          # uint16 tile-local row
        self.post_val = torch.empty(cap, dtype=torch.float64, device=dev)
        f32 = variant in ("dense32", "block")
        self.post_val32 = torch.empty(cap, dtype=torch.float32, device=dev) if f32 else None
        self.term_maxw = torch.empty(max(self.n_vocab, 1), dtype=torch.float32, device=dev) if variant == "dense32" else None
        self.post_pk = torch.empty((cap, 2), dtype=torch.int32, device=dev) if variant in ("block", "hash") else None   # {tile-local row, round(weight * 2^26)}
        self.csr = csr                                          # the to-matrix itself (exact re-scoring in dense32 / block)
        ws = _ws((ncell + 1) * 4 + 512 + _lib.load().pfz_scan_ws_bytes(ncell + 1))
        flags = 0
        if os.environ.get("PFZ_BANK_ORDER", "1") != "0" and variant != "hash":
            flags = 2 if f32 else 1                             # 32 four-byte banks for fp32 accumulators, 16 eight-byte banks for fp64
        _lib.call("pfz_index_build", _p(csr.indptr), _p(csr.indices), _p(csr.data), n, self.n_vocab, tile,
                  self.n_tiles, flags, _p(self.seg), _p(self.post_idx), _p(self.post_val), _p(self.post_val32), _p(self.term_maxw), _p(ws), _stream())
        if variant in ("block", "hash") and n > 0:
            if self.acc_bits == 16:                             # {word offset | half-word selector, w15}: what the 16-bit update consumes
                _lib.call("pfz_index_pack_q15", _p(self.post_idx), _p(self.post_val), ctypes.c_void_p(self.seg.data_ptr() + 4 * ncell), tile, _p(self.post_pk), _stream())
            else:
                _lib.call("pfz_index_pack_q26", _p(self.post_idx), _p(self.post_val), ctypes.c_void_p(self.seg.data_ptr() + 4 * ncell), _p(self.post_pk), _stream())


DENSE32_MAX_ROW_NNZ = 128


HASH_MIN_ROWS = int(os.environ.get("PFZ_HASH_MIN_ROWS", "32768"))   # below this the tile-based list kernel has few tiles to walk
HASH_MAX_ROW_NNZ = 256


def choose_variant(density, max_row_nnz=None, n_to=None):
    """K2 variant for an index: sparse inputs (density = postings visited per scored pair, NgramTfidf.density(), below
    DENSE_MIN_DENSITY) take the per-row hash kernel when the to-shard is large (work ~ postings) and the tile-walking
    `list` kernel otherwise; denser inputs take the dense-regime kernel.  The mixed-precision
    `dense32` filter needs its fp32 error bound (<= ~row_nnz * 2^-24) to stay below half its 2e-5 margin,
    so rows longer than DENSE32_MAX_ROW_NNZ n-grams select the plain fp64 `dense` kernel."""
    if density is None or density < DENSE_MIN_DENSITY:
        if (density is not None and n_to is not None and n_to >= HASH_MIN_ROWS and max_row_nnz is not None
                and max_row_nnz <= HASH_MAX_ROW_NNZ and SPARSE_VARIANT == "hash"):
            return "hash"
        return "list"
    if DENSE_VARIANT in ("dense32", "block") and (max_row_nnz is None or max_row_nnz > DENSE32_MAX_ROW_NNZ):
        return "dense"
    return DENSE_VARIANT


def index_for(csr_to, vec, index=None, tile=None):
    """The K2 index of the TF-IDF to-matrix csr_to for from-rows of up to vec.max_row_nnz terms.
    index=None: a new index of the variant choose_variant picks for the fitted vectoriser vec.  Otherwise `index` itself
    while its kernel takes rows that long; if not, a new index on index.csr for the fp64 kernel of the same regime: the
    block (and dense32) kernel holds 128 terms per row, the hash kernel 256, and both only flag a longer row on the device."""
    if index is None:
        return SparseIndex(csr_to, tile, variant=choose_variant(vec.density(), vec.max_row_nnz, csr_to.n_rows))
    if index.variant in ("dense32", "block") and vec.max_row_nnz > DENSE32_MAX_ROW_NNZ:
        return SparseIndex(index.csr, tile, variant="dense")
    if index.variant == "hash" and vec.max_row_nnz > HASH_MAX_ROW_NNZ:
        return SparseIndex(index.csr, tile, variant="list")
    return index


def _auto_splits(n_from, n_tiles, sm_count=132):
    want = sm_count * 32                                   # enough (from-row, tile-range) tasks to fill every SM
    if n_from >= want:
        return 1
    return max(1, min(n_tiles, (want + max(n_from, 1) - 1) // max(n_from, 1)))


K2_LIST, K2_DENSE, K2_DENSE32 = 1, 2, 3
DENSE_MIN_DENSITY = float(os.environ.get("PFZ_DENSE_MIN_DENSITY", "0.03"))
DENSE_VARIANT = os.environ.get("PFZ_DENSE_VARIANT", "block")     # which kernel serves the dense regime
SPARSE_VARIANT = os.environ.get("PFZ_SPARSE_VARIANT", "hash")    # ... and the sparse regime on large to-shards
K2_VARIANT = {"list": K2_LIST, "dense": K2_DENSE, "dense32": K2_DENSE32}
HASH_SLOTS = int(os.environ.get("PFZ_HASH_SLOTS", "0"))          # 0 = choose from the index


def _hash_slots(index):
    """Table size of the hash kernel.  2 048 slots (16 KB, 8 CTAs per SM; inherited, not re-tuned on H100) beat 8 192 and
    16 384 on the 1M x 1M uniform strings: rows that visit more postings take more
    passes over tile ranges, and a pass whose table fills is redone over halved to-row ranges inside the kernel."""
    return HASH_SLOTS if HASH_SLOTS else 2048
BLOCK_MAX_ROWS = (1 << 22) - 1                                   # row id field of the block kernel's clustering key


def _spcos_block(a, index, k, min_similarity, self_match, from_index_base, to_index_base, n_splits):
    """from-row-block kernel (pfz_spcos_topk_block): clustering + block tables + scoring, all enqueued on the stream."""
    dev = _dev()
    n_from = a.n_rows
    nnz_cap = int(a.indices.numel())
    ws = _ws(_lib.load().pfz_spcos_block_ws_bytes(n_from, nnz_cap, index.n_vocab, n_splits))
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    ti = torch.empty((n_splits, max(n_from, 1), k), dtype=torch.int32, device=dev)
    tv = torch.empty((n_splits, max(n_from, 1), k), dtype=torch.float64, device=dev)
    _lib.call("pfz_spcos_topk_block", _p(a.indptr), _p(a.indices), _p(a.data), n_from, nnz_cap, _p(index.seg), _p(index.post_pk),
              _p(index.csr.indptr), _p(index.csr.indices), _p(index.csr.data), index.n_vocab, index.tile, index.n_tiles, index.n_to, k,
              float(min_similarity), int(bool(self_match)), int(from_index_base), int(to_index_base), n_splits, BLOCK_ROWS, index.acc_bits, _p(ti), _p(tv), _p(err),
              _p(ws), _stream())
    if n_splits > 1:
        oi = torch.empty((max(n_from, 1), k), dtype=torch.int32, device=dev)
        ov = torch.empty((max(n_from, 1), k), dtype=torch.float64, device=dev)
        _lib.call("pfz_topk_merge", _p(ti), _p(tv), n_splits, n_from, k, k, _p(oi), _p(ov), _stream())
    else:
        oi, ov = ti[0], tv[0]
    return oi[:n_from], ov[:n_from], err


def spcos_topk(a: CsrMatrix, index: SparseIndex, k, min_similarity=0.0, self_match=False, from_index_base=0,
               to_index_base=0, n_splits=None, variant="auto"):
    """K2.  Returns (top_idx int32[n_from,k] GLOBAL to-indices or -1, top_val float64[n_from,k]) on device.
    variant: "list" | "dense" | "auto" (= the variant the index was tiled for, see choose_variant);
    both give identical results, they differ in cost model -- see pfz.h."""
    if variant == "auto":
        variant = index.variant
    dev = _dev()
    n_from = a.n_rows
    k = int(k)
    if k < 1:
        raise ValueError("top_n must be >= 1")
    if n_splits is None:
        n_splits = _auto_splits(n_from, index.n_tiles)
    n_splits = max(1, min(int(n_splits), index.n_tiles))
    if variant == "block":
        if index.post_pk is None:
            raise ValueError("the index was not built for the block variant")
        if k <= 32 and n_from <= BLOCK_MAX_ROWS:
            oi, ov, err = _spcos_block(a, index, k, min_similarity, self_match, from_index_base, to_index_base, n_splits)
            index._block_err = err                         # non-zero iff a from-row exceeded 128 terms (callers pick the variant so that it cannot)
            return oi, ov
        variant = "dense32"                                # paging (top_n > 32) runs on the per-row kernel over the same index
    counter = torch.zeros(n_splits, dtype=torch.int32, device=dev)
    if variant == "hash" and index.post_pk is None:
        raise ValueError("the index was not built for the hash variant")
    err = torch.zeros(1, dtype=torch.int32, device=dev) if variant == "hash" else None
    pages = []
    excl_v = excl_i = None
    remaining = k
    while remaining > 0:
        kp = min(32, remaining)
        ti = torch.empty((n_splits, max(n_from, 1), kp), dtype=torch.int32, device=dev)
        tv = torch.empty((n_splits, max(n_from, 1), kp), dtype=torch.float64, device=dev)
        if variant == "dense32" and index.post_val32 is None:
            raise ValueError("the index was not built for the dense32 variant")
        if variant == "hash":
            _lib.call("pfz_spcos_topk_hash", _p(a.indptr), _p(a.indices), _p(a.data), n_from, _p(index.seg), _p(index.post_pk),
                      _p(index.csr.indptr), _p(index.csr.indices), _p(index.csr.data), index.tile, index.n_tiles, index.n_to, kp,
                      float(min_similarity), int(bool(self_match)), int(from_index_base), int(to_index_base), n_splits, _hash_slots(index),
                      _p(excl_v), _p(excl_i), _p(ti), _p(tv), _p(counter), _p(err), _stream())
            index._hash_err = err                          # 2 = table overflow, 3 = row > 256 terms (choose_variant rules both out)
        else:
          _lib.call("pfz_spcos_topk", _p(a.indptr), _p(a.indices), _p(a.data), n_from, _p(index.seg), _p(index.post_idx),
                  _p(index.post_val), _p(index.post_val32), _p(index.csr.indptr), _p(index.csr.indices), _p(index.csr.data),
                  _p(index.term_maxw), index.n_vocab, index.tile, index.n_tiles, index.n_to, kp, float(min_similarity),
                  int(bool(self_match)), int(from_index_base), int(to_index_base), n_splits, _p(excl_v), _p(excl_i),
                  _p(ti), _p(tv), _p(counter), K2_VARIANT[variant], _stream())
        if n_splits > 1:
            oi = torch.empty((max(n_from, 1), kp), dtype=torch.int32, device=dev)
            ov = torch.empty((max(n_from, 1), kp), dtype=torch.float64, device=dev)
            _lib.call("pfz_topk_merge", _p(ti), _p(tv), n_splits, n_from, kp, kp, _p(oi), _p(ov), _stream())
        else:
            oi, ov = ti[0], tv[0]
        pages.append((oi, ov))
        remaining -= kp
        if remaining > 0:
            excl_v = ov[:, -1].contiguous(); excl_i = oi[:, -1].contiguous()
            # rows whose page is not full are exhausted: an idx of -1 disables the filter, so give them
            # an unbeatable exclusive key instead (nothing ranks after (-inf, INT_MAX))
            done = excl_i < 0
            excl_v = torch.where(done, torch.full_like(excl_v, float("-inf")), excl_v)
            excl_i = torch.where(done, torch.full_like(excl_i, 2 ** 31 - 1), excl_i)
    if len(pages) == 1:
        oi, ov = pages[0]
    else:
        oi = torch.cat([p[0] for p in pages], dim=1); ov = torch.cat([p[1] for p in pages], dim=1)
    return oi[:n_from], ov[:n_from]


def topk_merge(idx, val, k_out):
    """Merge [n_lists, n_from, k_in] candidate lists into the canonical top-k_out (device tensors)."""
    n_lists, n_from, k_in = idx.shape
    dev = idx.device
    oi = torch.empty((n_from, k_out), dtype=torch.int32, device=dev)
    ov = torch.empty((n_from, k_out), dtype=torch.float64, device=dev)
    _lib.call("pfz_topk_merge", _p(idx.contiguous()), _p(val.contiguous()), n_lists, n_from, k_in, k_out, _p(oi), _p(ov), _stream())
    return oi, ov
