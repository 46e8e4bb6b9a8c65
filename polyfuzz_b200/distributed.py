"""Multi-GPU plumbing: one process per GPU (torchrun), `torch.distributed` over NCCL/NVLink.

The path shards by to_list row-blocks (SURVEY.md section 8e): rank r owns to-rows
[r*ceil(n_to/G), ...), builds its own inverted index, scores every from-row against its shard with
GLOBAL to-indices, and the per-shard top-k lists are exchanged with ONE all-gather
(n_from * k * 16 B per rank) followed by the pfz_topk_merge kernel with the same
(score desc, index asc) key -- so the result is bit-identical to the single-GPU result.
tfidf_topk_sharded drives TF-IDF on one GPU too (comm=None: one shard, no collectives).
The TF-IDF fit needs the global vocabulary and document frequencies.  An n-gram code space of at most 2^24 takes one
all-reduce(SUM) of the dense int32 df table.  A larger one all-gathers the ranks' sorted local vocabularies (sum_r V_r * 8 B
received per rank), sorts the union on every rank, and all-reduces the int32 df indexed by global vocabulary rank (V * 4 B).
"""
import torch
import torch.distributed as dist


def shard_bounds(n_total, world_size, rank):
    """Contiguous row-block of rank: [lo, hi)."""
    per = (n_total + world_size - 1) // world_size if world_size > 0 else n_total
    lo = min(n_total, rank * per)
    return lo, min(n_total, lo + per)


def pack_topk(idx, val):
    """(int32[n,k], float64[n,k]) -> int64[n,k,2] so that one all-gather moves both."""
    buf = torch.empty(idx.shape + (2,), dtype=torch.int64, device=idx.device)
    buf[..., 0] = val.contiguous().view(torch.int64)
    buf[..., 1] = idx.to(torch.int64)
    return buf


def unpack_topk(buf):
    val = buf[..., 0].contiguous().view(torch.float64)
    idx = buf[..., 1].to(torch.int32).contiguous()
    return idx, val


class Comm:
    """Thin wrapper over a torch.distributed process group (nccl on GPUs, gloo in CPU tests)."""

    def __init__(self, group=None):
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialised (launch with torchrun)")
        self.group = group
        self.rank = dist.get_rank(group)
        self.world_size = dist.get_world_size(group)

    def all_reduce_sum(self, t):
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        return t

    def all_reduce_max(self, t):
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
        return t

    def all_gather_topk(self, idx, val):
        """-> (idx int32[G,n,k], val float64[G,n,k]); ONE collective."""
        local = pack_topk(idx, val)
        n = local.shape[0]
        out = torch.empty((self.world_size * n,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(out, local, group=self.group)        # concatenated along dim 0
        return unpack_topk(out.view((self.world_size, n) + tuple(local.shape[1:])))

    def all_gather_varlen(self, buf, n):
        """Variable-length all-gather of int64 buffers: this rank contributes buf[:n] (n: an int or a one-element tensor).
        -> (int64[G, L], [n_0, .., n_{G-1}] on the host): row r holds rank r's n_r entries followed by ~0 (-1) padding,
        L = max(max_r n_r, 1).  Two collectives (the lengths, then the buffers padded to the longest), one host read."""
        dev = buf.device
        mine = torch.as_tensor(n, dtype=torch.int64, device=dev).reshape(1)
        lens = torch.empty(self.world_size, dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(lens, mine, group=self.group)
        lengths = [int(x) for x in lens.tolist()]
        L = max(max(lengths), 1)
        local = torch.full((L,), -1, dtype=torch.int64, device=dev)
        local[:lengths[self.rank]] = buf[:lengths[self.rank]]
        out = torch.empty((self.world_size, L), dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(out.view(-1), local, group=self.group)
        return out, lengths


    def all_gather_best(self, idx, score, dist_):
        """Per-shard best matches (int32 idx[n] GLOBAL or -1, float64 score[n], int32 dist[n]) of every rank
        -> ([G,n], [G,n], [G,n]); ONE collective (the edit-distance matchers' exchange)."""
        n = idx.shape[0]
        local = torch.empty((n, 2), dtype=torch.int64, device=idx.device)
        local[:, 0] = score.contiguous().view(torch.int64)
        local[:, 1] = (idx.to(torch.int64) & 0xffffffff) | (dist_.to(torch.int64) << 32)
        out = torch.empty((self.world_size * n, 2), dtype=torch.int64, device=idx.device)
        dist.all_gather_into_tensor(out, local, group=self.group)
        out = out.view(self.world_size, n, 2)
        sc = out[..., 0].contiguous().view(torch.float64)
        lo32 = out[..., 1] & 0xffffffff
        gi = torch.where(lo32 >= 2 ** 31, lo32 - 2 ** 32, lo32).to(torch.int32).contiguous()
        gd = (out[..., 1] >> 32).to(torch.int32).contiguous()
        return gi, sc, gd


def merge_topk_any(idx, val, k_out):
    """Canonical merge of [G, n, k_in] per-shard lists into [n, k_out]: the pfz_topk_merge kernel up to 32, and for larger
    top_n two stable device sorts by the same key (score desc, index asc; empty slots last)."""
    from . import engine
    if k_out <= 32:
        return engine.topk_merge(idx, val, k_out)
    G, n, k_in = idx.shape
    ci = idx.permute(1, 0, 2).reshape(n, G * k_in)
    cv = val.permute(1, 0, 2).reshape(n, G * k_in)
    empty = ci < 0
    key_i = torch.where(empty, torch.full_like(ci, 2 ** 31 - 1), ci)
    o1 = torch.argsort(key_i, dim=1, stable=True)
    ci1, cv1, e1 = torch.gather(ci, 1, o1), torch.gather(cv, 1, o1), torch.gather(empty, 1, o1)
    key_v = torch.where(e1, torch.full_like(cv1, float("-inf")), cv1)
    o2 = torch.argsort(key_v, dim=1, descending=True, stable=True)
    oi = torch.gather(ci1, 1, o2)[:, :k_out].contiguous()
    ov = torch.gather(cv1, 1, o2)[:, :k_out].contiguous()
    ov = torch.where(oi < 0, torch.zeros_like(ov), ov)
    return oi, ov


def gather_string_shards(comm, S):
    """All-gather the ranks' device-resident to-list shards (engine.StagedStrings) into the whole list on every rank:
    -> (blob int32[n_chars_total], offsets int64[n_total + 1], all_ascii, None).  Two small collectives (sizes, then the padded
    byte blobs + offsets); used by the device frame tail (K5) so that no rank has to pack the other ranks' strings."""
    dev = S.d_off.device
    meta = torch.tensor([S.n_chars, S.n, int(bool(S.ascii))], dtype=torch.int64, device=dev)
    metas = torch.empty((comm.world_size, 3), dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(metas.view(-1), meta, group=comm.group)
    metas = metas.cpu()
    if int(metas[:, 2].min()) == 0:
        return (None, None, False, None)
    max_c, max_n = int(metas[:, 0].max()), int(metas[:, 1].max())
    loc_b = torch.zeros(max(max_c, 1), dtype=torch.uint8, device=dev)
    loc_b[:S.n_chars] = S.d_blob[:S.n_chars].to(torch.uint8)
    loc_o = torch.zeros(max_n + 1, dtype=torch.int64, device=dev)
    loc_o[:S.n + 1] = S.d_off[:S.n + 1]
    all_b = torch.empty((comm.world_size, loc_b.numel()), dtype=torch.uint8, device=dev)
    all_o = torch.empty((comm.world_size, max_n + 1), dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(all_b.view(-1), loc_b, group=comm.group)
    dist.all_gather_into_tensor(all_o.view(-1), loc_o, group=comm.group)
    blobs, offs, base = [], [], 0
    for r in range(comm.world_size):
        nc, nr = int(metas[r, 0]), int(metas[r, 1])
        blobs.append(all_b[r, :nc].to(torch.int32))
        offs.append(all_o[r, :nr] + base)
        base += nc
    offs.append(torch.tensor([base], dtype=torch.int64, device=dev))
    return (torch.cat(blobs) if base else torch.zeros(1, dtype=torch.int32, device=dev), torch.cat(offs), True, None)


def get_comm(group=None):
    """Comm for the default group, or None when not running distributed (world size 1)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        return Comm(group)
    return None


def tfidf_topk_sharded(vectorizer, staged_from, staged_to_shard, to_index_base, top_n, min_similarity,
                       self_match, from_index_base=0, fit=True, fit_on_from=True, comm=None, index=None,
                       tile=None, timings=None, k1_timings=None, n_docs_total=None):
    """TF-IDF top-k: K1, the K2 index (engine.index_for) and K2 -- the one driver of TFIDF.match, on one GPU (comm=None,
    the to-list is one shard at base 0) and on many.  Every rank passes the same from-list and its own to-shard; a
    single-GPU self-match passes the same StagedStrings as both, and one matrix serves both sides.
    fit=False transforms with the fitted vectoriser against `index`, which is replaced when the new from-rows are too long
    for its kernel; staged_from may then be an already vectorised from-matrix (engine.CsrMatrix).
    n_docs_total: the number of documents the fit counts over ALL ranks (to-rows of every shard + the from-list when
    fit_on_from), when the caller knows it -- saves one small all-reduce and a host sync per fit.
    Returns (top_idx[n_from,k] GLOBAL indices, top_val[n_from,k], csr_to_shard, index)."""
    from . import engine
    ev1 = None
    if k1_timings is not None:                              # K1 + index build, for bench.py's per-kernel breakdown
        ev1 = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev1[0].record()
    if fit:
        counted = [True, fit_on_from and (comm is None or comm.rank == 0)]
        staged = [staged_to_shard, staged_from]
        same = staged_from is staged_to_shard           # single-GPU self-match: one matrix for both sides
        if same:                                        # (polyfuzz/models/_tfidf.py:114-116)
            (rows_to,) = vectorizer.fit_staged([staged_to_shard], comm=comm, n_docs_total=n_docs_total)
            rows_from = rows_to
        else:
            rows_to, rows_from = vectorizer.fit_staged(staged, counted=counted, comm=comm, n_docs_total=n_docs_total)
        csr_to = vectorizer.emit(rows_to)
        index = engine.index_for(csr_to, vectorizer, tile=tile)
        csr_from = csr_to if same else vectorizer.emit(rows_from)
    else:
        csr_to = None
        if isinstance(staged_from, engine.CsrMatrix):       # already vectorised (a self-match transform on one GPU)
            csr_from = staged_from
        else:
            csr_from = vectorizer.emit(vectorizer.rows(staged_from))
        index = engine.index_for(index.csr, vectorizer, index, tile)
    if ev1 is not None:
        ev1[1].record()
        k1_timings.append(ev1)
    ev = None
    if timings is not None:
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    idx, val = engine.spcos_topk(csr_from, index, top_n, min_similarity, self_match=self_match,
                                 from_index_base=from_index_base, to_index_base=to_index_base)
    if ev is not None:
        ev[1].record()
        timings.append(ev)
    if comm is not None:
        gi, gv = comm.all_gather_topk(idx.contiguous(), val.contiguous())
        idx, val = merge_topk_any(gi, gv, top_n)
    return idx, val, csr_to, index
