"""Multi-GPU TF-IDF fit with an n-gram code space above 2^24 (no dense df table): the ranks' sorted local vocabularies are
all-gathered, every rank sorts their union, and the df indexed by global vocabulary rank is all-reduced (DESIGN.md section 5).

On one GPU the ranks run as threads that talk through an in-process communicator; every rank's vocabulary, df, idf, CSR
shard and the merged top-k must equal the single-GPU fit bit for bit.  With two GPUs or more, tools/dist_vocab_check.py runs
the same comparison over NCCL on whole frames.  The variable-length all-gather itself is tested over gloo on the CPU."""
import os
import pickle
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
gpu = pytest.mark.gpu


# ---- an in-process communicator: G rank threads on one GPU, one stream -------------------------------------------------------
class _Hub:
    def __init__(self, G):
        self.G = G
        self.barrier = threading.Barrier(G, timeout=120)     # a protocol error fails the test instead of hanging it
        self.turn = threading.Lock()                         # one rank runs host code at a time, the others wait in a collective
        self.slots = [None] * G


class FakeComm:
    """The collectives of distributed.Comm, done in process on device tensors.  Every rank enqueues on the same (default)
    stream, so a rank's reads of the other ranks' tensors are ordered after the work that wrote them."""

    def __init__(self, hub, rank):
        self.hub, self.rank, self.world_size = hub, rank, hub.G

    def _wait(self):
        self.hub.turn.release()
        try:
            self.hub.barrier.wait()
        finally:
            self.hub.turn.acquire()

    def _exchange(self, t):
        self.hub.slots[self.rank] = t
        self._wait()
        got = list(self.hub.slots)
        self._wait()                                         # every rank has read the slots before the next exchange writes them
        return got

    def all_reduce_sum(self, t):
        t.copy_(torch.stack(self._exchange(t.clone())).sum(0).to(t.dtype))
        return t

    def all_reduce_max(self, t):
        t.copy_(torch.stack(self._exchange(t.clone())).amax(0))
        return t

    def all_gather_topk(self, idx, val):
        got = self._exchange((idx.clone(), val.clone()))
        return torch.stack([g[0] for g in got]), torch.stack([g[1] for g in got])

    def all_gather_varlen(self, buf, n):
        n = int(torch.as_tensor(n).reshape(-1)[0])
        got = self._exchange(buf[:n].clone())
        lengths = [g.numel() for g in got]
        out = torch.full((self.world_size, max(max(lengths), 1)), -1, dtype=torch.int64, device=buf.device)
        for r, g in enumerate(got):
            out[r, :g.numel()] = g
        return out, lengths


def run_ranks(G, fn):
    """fn(comm) on G rank threads -> (results, exceptions), one per rank."""
    hub = _Hub(G)
    res, err = [None] * G, [None] * G

    def body(r):
        torch.cuda.set_device(0)
        with hub.turn:
            try:
                res[r] = fn(FakeComm(hub, r))
            except BaseException as e:                       # noqa: BLE001 -- reported per rank below
                err[r] = e
                hub.barrier.abort()                          # ranks still waiting in a collective fail now
    threads = [threading.Thread(target=body, args=(r,)) for r in range(G)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in threads), "a rank thread did not finish"
    return res, err


def run_ok(G, fn):
    res, err = run_ranks(G, fn)
    for r, e in enumerate(err):
        if e is not None:
            raise AssertionError(f"rank {r} raised {e!r}") from e
    return res


# ---- single-GPU and sharded fits ------------------------------------------------------------------------------------------------
def _state(v, csr):
    return dict(keys=np.asarray(v.vocab_keys).copy(), df=np.asarray(v.df).copy(), idf=np.asarray(v.idf).copy(), csr=csr.to_scipy())


def single(frm, to, rng, clean, k, from_block=None):
    """The single-GPU matcher: (state of its fit, top-k idx, val, the k it used)."""
    import polyfuzz_b200
    m = polyfuzz_b200.TFIDF(n_gram_range=rng, clean_string=clean, min_similarity=0.0, top_n=k)
    idx, val, kk = m.match_arrays(frm, to, from_block=from_block)
    return m, _state(m.vectorizer, m.tf_idf_to), idx.cpu(), val.cpu(), kk


def sharded(comm, frm, to, rng, clean, k, from_block=None, n_docs_total=True):
    """What TFIDF.match_arrays does on one rank, without the string exchange of the frame tail."""
    from polyfuzz_b200 import engine
    from polyfuzz_b200.distributed import shard_bounds, tfidf_topk_sharded
    v = engine.NgramTfidf(rng, clean, True)
    self_match = to is None
    full_to = to if to else frm
    base, rows = 0, frm
    if from_block is not None:
        base, rows = from_block[0], frm[from_block[0]:from_block[1]]
    lo, hi = shard_bounds(len(full_to), comm.world_size, comm.rank)
    n_docs = len(full_to) + (len(rows) if to else 0)
    idx, val, csr, index = tfidf_topk_sharded(v, v.stage(rows), v.stage(full_to[lo:hi]), lo, k, 0.0, self_match, base,
                                              fit_on_from=bool(to), comm=comm, n_docs_total=n_docs if n_docs_total else None)
    return dict(_state(v, csr), idx=idx.cpu(), val=val.cpu(), lo=lo, hi=hi, v=v, index=index, csr_dev=csr)


def assert_rank_equals_single(r, ref, idx, val):
    assert r["keys"].dtype == np.uint64 and np.array_equal(r["keys"], ref["keys"])
    assert np.array_equal(r["df"], ref["df"])
    assert np.array_equal(r["idf"].view(np.int64), ref["idf"].view(np.int64))
    lo, hi = r["lo"], r["hi"]
    want = ref["csr"][lo:hi]
    got = r["csr"]
    assert got.shape == want.shape
    assert np.array_equal(got.indptr, want.indptr)
    assert np.array_equal(got.indices, want.indices)
    assert np.array_equal(got.data.view(np.int64), want.data.view(np.int64))
    assert torch.equal(r["idx"], idx) and torch.equal(r["val"].view(torch.int64), val.view(torch.int64))


@pytest.fixture(scope="module")
def titles():
    from polyfuzz_b200 import synth
    to = synth.titles(2500, seed=31)
    frm = synth.titles(700, seed=32) + ["", "x", "Ünïcødé Çafé", to[3]]
    return frm, to


def _large(rng, clean, strings):
    from polyfuzz_b200 import engine
    v = engine.NgramTfidf(rng, clean, True)
    v.fit(strings)
    return v.code_space() > engine.DENSE_CODE_SPACE_MAX


# ---- one GPU, emulated ranks ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("G", [2, 3, 4])
@pytest.mark.parametrize("rng,clean,large", [((3, 6), True, True), ((2, 5), True, True), ((1, 3), False, False), ((3, 4), False, True)])
def test_two_lists_equal_single_gpu(titles, rng, clean, large, G):
    """The configurations of the single-GPU large code space test; raw (1, 3) on these titles ((alphabet + 1)^3 < 2^24)
    keeps the dense df table."""
    frm, to = titles
    assert _large(rng, clean, to + frm) == large
    _, ref, idx, val, k = single(frm, to, rng, clean, 5)
    for r in run_ok(G, lambda c: sharded(c, frm, to, rng, clean, k)):
        assert_rank_equals_single(r, ref, idx, val)


@gpu
@pytest.mark.parametrize("G", [2, 3])
def test_raw_trigrams_over_many_code_points(G):
    """Raw (3, 3) on a list of more than 255 distinct code points (CJK): 401^3 > 2^24, and the document count is all-reduced
    (no n_docs_total)."""
    g = np.random.default_rng(7)
    cjk = [chr(0x4E00 + i) for i in range(400)]
    words = ["".join(g.choice(cjk, g.integers(2, 5))) for _ in range(600)]
    to = [" ".join(g.choice(words, g.integers(1, 4))) for _ in range(1500)]
    frm = [" ".join(g.choice(words, g.integers(1, 4))) for _ in range(300)] + [to[0], "abc 東京"]
    assert _large((3, 3), False, to + frm)
    _, ref, idx, val, k = single(frm, to, (3, 3), False, 4)
    for r in run_ok(G, lambda c: sharded(c, frm, to, (3, 3), False, k, n_docs_total=False)):
        assert_rank_equals_single(r, ref, idx, val)


@gpu
@pytest.mark.parametrize("G", [2, 4])
def test_self_match_and_from_block(titles, G):
    _, to = titles
    names = to[:1800]
    _, ref, idx, val, k = single(names, None, (3, 6), True, 6)
    for r in run_ok(G, lambda c: sharded(c, names, None, (3, 6), True, k)):
        assert_rank_equals_single(r, ref, idx, val)
    _, ref, idx, val, k = single(names, None, (3, 4), False, 6, from_block=(500, 1100))
    for r in run_ok(G, lambda c: sharded(c, names, None, (3, 4), False, k, from_block=(500, 1100))):
        assert_rank_equals_single(r, ref, idx, val)


@gpu
def test_empty_shard_and_empty_local_vocabulary(titles):
    frm, to = titles
    # 3 to-strings over 4 ranks: the last rank's shard is empty (its local vocabulary too)
    small_to, small_frm = to[:3], frm[:50]
    _, ref, idx, val, k = single(small_frm, small_to, (3, 6), True, 3)
    res = run_ok(4, lambda c: sharded(c, small_frm, small_to, (3, 6), True, k))
    assert res[3]["hi"] == res[3]["lo"]
    for r in res:
        assert_rank_equals_single(r, ref, idx, val)
    # the second of two ranks owns only strings shorter than the n-gram range, and is not the rank that counts the from-list
    short_to = to[:6] + ["ab", "", "x y", "!!!!!!!!", "a", "--"]
    for frm_, to_ in ((frm[:40], short_to), (short_to, None)):
        _, ref, idx, val, k = single(frm_, to_, (3, 5), True, 2)
        res = run_ok(2, lambda c: sharded(c, frm_, to_, (3, 5), True, k))
        assert res[1]["csr"].nnz == 0
        for r in res:
            assert_rank_equals_single(r, ref, idx, val)


@gpu
@pytest.mark.parametrize("n_docs_total", [True, False])
def test_all_strings_too_short_raise_on_every_rank(n_docs_total):
    import polyfuzz_b200
    to, frm = ["a", "!!!!!!!", "bc", "-- --", "x"], ["#####", "ab"]
    with pytest.raises(ValueError, match="empty vocabulary"):
        polyfuzz_b200.TFIDF(n_gram_range=(3, 6), min_similarity=0.0).match(frm, to)
    _, err = run_ranks(3, lambda c: sharded(c, frm, to, (3, 6), True, 1, n_docs_total=n_docs_total))
    for e in err:
        assert isinstance(e, ValueError) and "empty vocabulary" in str(e), err


@gpu
@pytest.mark.parametrize("rng,clean", [((3, 5), True), ((3, 4), False)])
def test_transform_after_sharded_fit_and_after_pickle(titles, rng, clean):
    """re_train=False: a new from-list against each rank's kept index, directly and after a pickle round trip of the fitted
    vectoriser and the rank's CSR shard (the index is rebuilt from it, as TFIDF does after unpickling)."""
    from polyfuzz_b200 import engine
    from polyfuzz_b200.distributed import tfidf_topk_sharded
    frm, to = titles
    new = frm[200:500] + ["Ünïcødé Çafé", "zz", "", to[10]]
    m, _, _, _, k = single(frm, to, rng, clean, 4)
    idx, val, _ = m.match_arrays(new, to, re_train=False)
    idx, val = idx.cpu(), val.cpu()

    def rank(comm):
        r = sharded(comm, frm, to, rng, clean, k)
        out = []
        v, index = r["v"], r["index"]
        for again in (False, True):
            if again:
                v = pickle.loads(pickle.dumps(v))
                csr = engine.CsrMatrix.from_scipy(r["csr_dev"].to_scipy())
                index = engine.SparseIndex(csr, variant=engine.choose_variant(v.density(), v.max_row_nnz, csr.n_rows))
            i, s, _, index = tfidf_topk_sharded(v, v.stage(new), None, r["lo"], k, 0.0, False, fit=False, comm=comm, index=index)
            out.append((i.cpu(), s.cpu()))
        return out
    for per_rank in run_ok(3, rank):
        for i, s in per_rank:
            assert torch.equal(i, idx) and torch.equal(s.view(torch.int64), val.view(torch.int64))


@gpu
@pytest.mark.parametrize("rng,large", [((3, 3), False), ((3, 5), True)])
def test_new_entry_point_only_on_the_large_code_space_path(titles, monkeypatch, rng, large):
    """Code space <= 2^24 keeps the dense df all-reduce and never calls pfz_df_scatter; above it, the new path runs."""
    from polyfuzz_b200 import _lib
    frm, to = titles
    names, lock = [], threading.Lock()
    real = _lib.call

    def record(name, *args):
        with lock:
            names.append(name)
        return real(name, *args)
    monkeypatch.setattr(_lib, "call", record)
    _, ref, idx, val, k = single(frm, to, rng, True, 3)
    assert ("pfz_df_dense" in names) != large and "pfz_df_scatter" not in names
    names.clear()
    for r in run_ok(2, lambda c: sharded(c, frm, to, rng, True, k)):
        assert_rank_equals_single(r, ref, idx, val)
    assert ("pfz_df_scatter" in names) == large
    assert ("pfz_df_dense" in names) != large


# ---- two GPUs or more, NCCL ----------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_nccl_frames_equal_single_gpu():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(29900 + os.getpid() % 90), os.path.join(ROOT, "tools", "dist_vocab_check.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert "DIST_VOCAB_CHECK PASS" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]


# ---- CPU, gloo, world size 2: the variable-length all-gather -------------------------------------------------------------------
def _varlen_worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from polyfuzz_b200.distributed import get_comm
        comm = get_comm()
        big = [-2, 2 ** 63 - 1, -(2 ** 63), 5, 0, 7]                 # uint64 codes >= 2^63 travel as negative int64
        cases = [([3, 1, 4, 1, 5], [9, 2]), ([], [8, 8, 8]), (big, []), ([], [])]
        for mine0, mine1 in cases:
            mine = (mine0, mine1)[rank]
            buf = torch.tensor(mine + [123, 456], dtype=torch.int64)   # entries past n are not sent
            n = torch.tensor([len(mine)], dtype=torch.int32)
            got, lengths = comm.all_gather_varlen(buf, n)
            L = max(len(mine0), len(mine1), 1)
            assert lengths == [len(mine0), len(mine1)], lengths
            want = [m + [-1] * (L - len(m)) for m in (mine0, mine1)]
            assert got.dtype == torch.int64 and got.tolist() == want, (got, want)
            got2, lengths2 = comm.all_gather_varlen(buf, len(mine))    # a host int works as the length too
            assert torch.equal(got2, got) and lengths2 == lengths
        out.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        out.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_all_gather_varlen_gloo():
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = 31500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_varlen_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = [out.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res
