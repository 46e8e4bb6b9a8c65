"""K2 (sparse cosine top-n) at ties and thresholds, on every kernel variant, compared with == against the oracle
(oracle/spdot_topn.c: indices and fp64 scores).

The kernels reach the contract -- keep a pair iff score > min_similarity, rank by (score desc, index asc), empty slots
(-1, 0.0) -- through approximate gates that differ per variant; a mistake in one of them loses or reorders entries only at a
tie or at the threshold.  tests/k2_cases.py builds exactly those inputs: runs of identical to-strings across to-tile, tile
split, shard, 16-bit accumulator word and 32-entry page boundaries, identical from-rows across block boundaries, and
min_similarity values equal to attained scores (and the doubles next to them)."""
import math

import numpy as np
import pytest
import torch

import k2_cases as kc
from oracle import native as onative
from oracle import tfidf as otfidf
from oracle.assemble import assemble as oracle_assemble

pytestmark = pytest.mark.gpu

# (index variant, block accumulator bits, block rows per CTA, hash table slots)
CONFIGS = {"list": ("list", 16, 8, 0), "dense": ("dense", 16, 8, 0), "dense32": ("dense32", 16, 8, 0)}
CONFIGS.update({f"block{b}x{r}": ("block", b, r, 0) for b in (16, 32) for r in (4, 8, 16)})
CONFIGS.update({f"hash{h}": ("hash", 16, 8, h) for h in (1024, 2048, 8192, 16384)})
MODES = ("two", "self")


@pytest.fixture(scope="module")
def pf():
    import polyfuzz_b200
    from polyfuzz_b200 import engine
    return polyfuzz_b200, engine


def _force_variant(monkeypatch, engine, variant):
    monkeypatch.setattr(engine, "DENSE_MIN_DENSITY", 1e9 if variant == "list" else 0.0)
    monkeypatch.setattr(engine, "DENSE_VARIANT", variant if variant != "list" else "dense")
    if variant != "block":                                             # (the block kernel's tables hold <= 128 terms per row)
        monkeypatch.setattr(engine, "DENSE32_MAX_ROW_NNZ", 1 << 30)    # exercise the filter even on long rows


def _configure(monkeypatch, engine, name):
    variant, bits, rows, slots = CONFIGS[name]
    monkeypatch.setattr(engine, "BLOCK_ACC_BITS", bits)
    monkeypatch.setattr(engine, "BLOCK_ROWS", rows)
    monkeypatch.setattr(engine, "HASH_SLOTS", slots)
    return variant, bits


def _tiles(name):
    variant, bits, _, _ = CONFIGS[name]
    return kc.TILES[f"block{bits}" if variant == "block" else variant]


class _Gpu:
    """The tie case on the device: CSRs from the GPU vectoriser (checked against the oracle vectoriser), indexes and
    oracle lists made once and shared by every test of the module."""

    def __init__(self, engine):
        self.engine = engine
        self.case = kc.TieCase()
        self.dev, self.host, self._ix, self._or = {}, {}, {}, {}
        for mode in MODES:
            v = engine.NgramTfidf((3, 3), True, True)
            if mode == "self":
                (rows,) = v.fit_rows([self.case.to])
                csr_f = csr_t = v.emit(rows)
            else:
                rows_t, rows_f = v.fit_rows([self.case.to, self.case.frm])
                csr_t, csr_f = v.emit(rows_t), v.emit(rows_f)
            f, t = csr_f.to_scipy(), csr_t.to_scipy()
            of, ot = kc.canonical_vectors(self.case, mode)
            for got, exp in ((f, of), (t, ot)):
                np.testing.assert_array_equal(got.indptr, exp.indptr)
                np.testing.assert_array_equal(got.indices, exp.indices)
                np.testing.assert_array_equal(got.data, exp.data)
            self.dev[mode] = (csr_f, csr_t)
            self.host[mode] = (f, t)
        self.runs, self.ths = {}, {}
        for mode in MODES:
            oi, ov = self.oracle(mode, 0.0)
            src = self.case.from_list(mode)
            self.runs[mode] = [kc.run_score(oi, ov, src.index(self.case.var[f]), self.case.run_pos[f]) for f in range(len(kc.HEADS))]
            self.ths[mode] = kc.thresholds(oi, ov, self.runs[mode])[1]

    def index(self, mode, variant, tile, bits):
        key = (mode, variant, tile, bits)
        if key not in self._ix:
            self._ix[key] = self.engine.SparseIndex(self.dev[mode][1], tile=tile, variant=variant)
        return self._ix[key]

    def oracle(self, mode, ms):
        key = (mode, ms)
        if key not in self._or:
            f, t = self.host[mode]
            self._or[key] = onative.spdot_topn(f, t, kc.K_MAX, ms, self_match=mode == "self", n_threads=8)
        return self._or[key]

    def self_score(self, mode):
        f, _ = self.host[mode]
        return kc.self_scores(f[self.case.identical_from_rows(mode)[:1]])[0]


@pytest.fixture(scope="module")
def gpu(pf):
    return _Gpu(pf[1])


def _assert_no_err(ix, what):
    """The block / hash kernels flag a broken contract (a row over their term cap, a full hash table) on the device."""
    if getattr(ix, "_block_err", None) is not None:
        assert int(ix._block_err.item()) == 0, what
    if getattr(ix, "_hash_err", None) is not None:
        assert int(ix._hash_err.item()) == 0, what


def _check(ix, idx, val, oi, ov, what):
    _assert_no_err(ix, what)
    gi, gv = idx.cpu().numpy(), val.cpu().numpy()
    bad = np.nonzero((gi != oi).any(1) | (gv != ov).any(1))[0]
    assert len(bad) == 0, f"{what}: {len(bad)} rows differ, first {bad[:5].tolist()}: got {gi[bad[0]].tolist()} " \
                          f"{gv[bad[0]].tolist()} want {oi[bad[0]].tolist()} {ov[bad[0]].tolist()}"


def _reset_err(ix):
    ix._block_err = ix._hash_err = None


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("mode", MODES)
def test_tied_runs_across_tiles_splits_and_pages(pf, gpu, monkeypatch, name, mode):
    """ms = 0, every k of KS, the smallest legal tile and larger ones, n_splits 1, 2 and n_tiles: the runs of identical
    to-rows sit on the tile and split boundaries and cross ranks 31/32 and 63/64; identical from-rows agree."""
    _, engine = pf
    variant, bits = _configure(monkeypatch, engine, name)
    f, _ = gpu.dev[mode]
    oi, ov = gpu.oracle(mode, 0.0)
    ident = gpu.case.identical_from_rows(mode)
    for tile in _tiles(name):
        ix = gpu.index(mode, variant, tile, bits)
        assert ix.tile == kc.index_tile(variant, gpu.case.n_to, tile, bits)
        for n_splits in sorted({1, 2, ix.n_tiles}):
            for k in kc.KS:
                _reset_err(ix)
                idx, val = engine.spcos_topk(f, ix, k, 0.0, self_match=mode == "self", n_splits=n_splits)
                _check(ix, idx, val, oi[:, :k], ov[:, :k], f"{name} {mode} tile={ix.tile} n_splits={n_splits} k={k}")
                kc.assert_identical_rows_agree(idx.cpu().numpy(), val.cpu().numpy(), ident, mode == "self", k,
                                               self_score=gpu.self_score(mode))


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("mode", MODES)
def test_thresholds_at_attained_scores(pf, gpu, monkeypatch, name, mode):
    """min_similarity on attained scores (a tied run's score, the most frequent and the median score), the doubles next to
    them, 1.0 (duplicates score above it by an ulp), the double below 1.0 (single-n-gram rows score exactly 1.0) and a
    negative value; the smallest tile, one split and one per tile."""
    _, engine = pf
    variant, bits = _configure(monkeypatch, engine, name)
    f, _ = gpu.dev[mode]
    ix = gpu.index(mode, variant, _tiles(name)[0], bits)
    for ms in gpu.ths[mode]:
        oi, ov = gpu.oracle(mode, ms)
        for n_splits in sorted({1, ix.n_tiles}):
            for k in (1, 7, 33, 70):
                _reset_err(ix)
                idx, val = engine.spcos_topk(f, ix, k, ms, self_match=mode == "self", n_splits=n_splits)
                _check(ix, idx, val, oi[:, :k], ov[:, :k], f"{name} {mode} ms={ms!r} n_splits={n_splits} k={k}")


@pytest.mark.parametrize("name", list(CONFIGS))
def test_shards_with_index_bases(pf, gpu, monkeypatch, name):
    """The to-list in 2 and 3 shards (to_index_base = shard start), merged with engine.topk_merge (k <= 32) or
    distributed.merge_topk_any; the self-match scores a from-block that straddles a shard boundary (from_index_base)."""
    _, engine = pf
    from polyfuzz_b200.distributed import merge_topk_any, shard_bounds
    variant, bits = _configure(monkeypatch, engine, name)
    tile = _tiles(name)[0]
    n = gpu.case.n_to
    for mode in MODES:
        f_all, t_all = gpu.host[mode]
        for g in kc.SHARDS:
            b = shard_bounds(n, g, 1)[0]
            flo, fhi = (b - 400, b + 300) if mode == "self" else (0, f_all.shape[0])
            f_blk = f_all[flo:fhi]
            f_dev = engine.CsrMatrix.from_scipy(f_blk)
            shards = [shard_bounds(n, g, r) for r in range(g)]
            ixs = [engine.SparseIndex(engine.CsrMatrix.from_scipy(t_all[lo:hi]), tile=tile, variant=variant) for lo, hi in shards]
            for ms in (0.0, gpu.runs[mode][1], math.nextafter(gpu.runs[mode][1], -math.inf)):
                oi, ov = onative.spdot_topn(f_blk, t_all, kc.K_MAX, ms, self_match=mode == "self", from_index_base=flo, n_threads=8)
                for k in (1, 7, 32, 33, 70):
                    what = f"{name} {mode} shards={g} ms={ms!r} k={k}"
                    parts_i, parts_v = [], []
                    for (lo, _), ix in zip(shards, ixs):
                        _reset_err(ix)
                        i_, v_ = engine.spcos_topk(f_dev, ix, k, ms, self_match=mode == "self", from_index_base=flo, to_index_base=lo)
                        _assert_no_err(ix, what)
                        parts_i.append(i_); parts_v.append(v_)
                    si, sv = torch.stack(parts_i), torch.stack(parts_v)
                    mi, mv = engine.topk_merge(si, sv, k) if k <= 32 else merge_topk_any(si, sv, k)
                    _check(ix, mi, mv, oi[:, :k], ov[:, :k], what)


# ---- merges -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_lists,k_in,k_out", [(3, 5, 7), (4, 12, 32), (2, 40, 32), (3, 33, 5), (5, 32, 1), (2, 7, 32), (6, 3, 12)])
def test_topk_merge_kernel_on_crafted_lists(pf, n_lists, k_in, k_out):
    """Cross-list ties, (-1, 0.0) slots anywhere in a list, k_in below and above k_out and above 32."""
    _, engine = pf
    idx, val = kc.crafted_merge_lists(n_lists, 300, k_in, seed=11 * k_in + k_out)
    oi, ov = onative.topk_merge(idx, val, k_out)
    mi, mv = engine.topk_merge(torch.from_numpy(idx).cuda(), torch.from_numpy(val).cuda(), k_out)
    np.testing.assert_array_equal(mi.cpu().numpy(), oi)
    np.testing.assert_array_equal(mv.cpu().numpy(), ov)


@pytest.mark.parametrize("n_lists,k_in,k_out", [(2, 40, 33), (3, 33, 70), (1, 70, 70), (4, 12, 33), (3, 20, 32)])
def test_merge_topk_any_on_crafted_lists(pf, n_lists, k_in, k_out):
    """merge_topk_any: the kernel up to 32, the two stable sorts above."""
    from polyfuzz_b200.distributed import merge_topk_any
    idx, val = kc.crafted_merge_lists(n_lists, 300, k_in, seed=13 * k_in + k_out)
    oi, ov = onative.topk_merge(idx, val, k_out)
    mi, mv = merge_topk_any(torch.from_numpy(idx).cuda(), torch.from_numpy(val).cuda(), k_out)
    np.testing.assert_array_equal(mi.cpu().numpy(), oi)
    np.testing.assert_array_equal(mv.cpu().numpy(), ov)


def test_topk_merge_kernel_refuses_k_out_above_32(pf):
    _, engine = pf
    idx, val = kc.crafted_merge_lists(2, 10, 20, seed=1)
    with pytest.raises(RuntimeError, match="k_out=33"):
        engine.topk_merge(torch.from_numpy(idx).cuda(), torch.from_numpy(val).cuda(), 33)


# ---- row-size switches --------------------------------------------------------------------------------------------
def _frame_eq(df, ref):
    assert list(df.columns) == list(ref.columns)
    for c in df.columns:
        if c.startswith("Similarity"):
            np.testing.assert_array_equal(df[c].to_numpy(), ref[c].to_numpy())
        else:
            assert [None if (isinstance(v, float) and np.isnan(v)) else v for v in df[c].tolist()] == \
                   [None if (isinstance(v, float) and np.isnan(v)) else v for v in ref[c].tolist()], c


def _switch_lists(n, seed):
    """A to-list of short rows that also holds every trigram of a string of n distinct trigrams (in pieces of <= 64), and
    from-lists with and without that string."""
    from polyfuzz_b200 import synth
    long = kc.distinct_trigram_string(n, seed)
    pieces = [long[i:i + 66] for i in range(0, len(long) - 2, 64)]
    to = synth.company_names(3000, seed=seed) + pieces + pieces
    frm = synth.company_names(400, seed=seed + 1)
    new = synth.company_names(200, seed=seed + 2) + [long, long[:100], pieces[0]]
    return long, to, frm, new


@pytest.mark.parametrize("n,regime,short_variant,long_variant", [(128, "dense", "block", "block"), (129, "dense", "block", "dense"),
                                                                 (256, "sparse", "hash", "hash"), (257, "sparse", "hash", "list")])
def test_variant_switch_at_row_size(pf, monkeypatch, n, regime, short_variant, long_variant):
    """Rows of 128 / 129 distinct trigrams keep / leave the block index (its tables hold 128 terms per row), rows of
    256 / 257 keep / leave the hash index: through TFIDF.match, through match(..., re_train=False) after a fit on short rows,
    and through the sharded driver's transform path."""
    polyfuzz_b200, engine = pf
    from polyfuzz_b200.distributed import tfidf_topk_sharded
    if regime == "dense":
        monkeypatch.setattr(engine, "DENSE_MIN_DENSITY", 0.0)
        monkeypatch.setattr(engine, "DENSE_VARIANT", "block")
    else:
        monkeypatch.setattr(engine, "DENSE_MIN_DENSITY", 1e9)
        monkeypatch.setattr(engine, "SPARSE_VARIANT", "hash")
        monkeypatch.setattr(engine, "HASH_MIN_ROWS", 1)
    long, to, frm, new = _switch_lists(n, seed=n)
    # fit with the long row in the from-list
    m = polyfuzz_b200.TFIDF(min_similarity=0.0, top_n=7)
    idx, val, k = m.match_arrays(frm + [long], to)
    assert m._index.variant == long_variant
    f, t, _ = otfidf.fit_transform_sklearn(frm + [long], to)
    oi, ov = onative.spdot_topn(f, t, k, 0.0, n_threads=8)
    np.testing.assert_array_equal(idx.cpu().numpy(), oi)
    np.testing.assert_array_equal(val.cpu().numpy(), ov)
    # fit on short rows, then transform the long one
    m = polyfuzz_b200.TFIDF(min_similarity=0.0, top_n=7)
    m.match(frm, to)
    assert m._index.variant == short_variant
    got = m.match(new, to, re_train=False)
    assert m._index.variant == long_variant
    o = otfidf.TfidfOracle().fit(list(to) + list(frm))
    assert o.transform([long]).indptr[1] == n
    oi, ov = onative.spdot_topn(o.transform(new), o.transform(to), 7, 0.0, n_threads=8)
    _frame_eq(got, oracle_assemble(new, to, oi, ov))
    # the sharded driver (one rank): fit, then a transform-only call on the same index
    vec = engine.NgramTfidf((3, 3), True, True)
    _, _, _, ix = tfidf_topk_sharded(vec, vec.stage(frm), vec.stage(to), 0, 7, 0.0, False)
    assert ix.variant == short_variant
    i2, v2, _, ix2 = tfidf_topk_sharded(vec, vec.stage(new), None, 0, 7, 0.0, False, fit=False, index=ix)
    assert ix2.variant == long_variant
    np.testing.assert_array_equal(i2.cpu().numpy(), oi)
    np.testing.assert_array_equal(v2.cpu().numpy(), ov)


def test_k1_long_row_at_8192_slots_bit_exact(pf):
    """A string of exactly 8 192 trigram slots (the long-row kernel's limit) vectorises bit for bit as the oracle does."""
    _, engine = pf
    from polyfuzz_b200 import synth
    s = kc.string_with_slots(8192, (3, 3), seed=5)
    to = synth.company_names(300, seed=6) + [s, s[:3000]]
    frm = [s, s[:8000], "abc"] + synth.company_names(50, seed=7)
    v = engine.NgramTfidf((3, 3), True, True)
    rows_to, rows_from = v.fit_rows([to, frm])
    f, t, _ = otfidf.fit_transform_sklearn(frm, to)
    for got, exp in ((v.emit(rows_to).to_scipy(), t), (v.emit(rows_from).to_scipy(), f)):
        np.testing.assert_array_equal(got.indptr, exp.indptr)
        np.testing.assert_array_equal(got.indices, exp.indices)
        np.testing.assert_array_equal(got.data, exp.data)


@pytest.mark.parametrize("rng", [(3, 3), (3, 4)])
def test_k1_refuses_8193_slots(pf, rng):
    polyfuzz_b200, engine = pf
    s = kc.string_with_slots(8193, rng, seed=8)
    with pytest.raises(ValueError, match="at most 8192"):
        engine.NgramTfidf(rng, True, True).fit_rows([["abc def", s]])
    with pytest.raises(ValueError, match="at most 8192"):
        polyfuzz_b200.TFIDF(n_gram_range=rng, min_similarity=0.0).match(["abc def"], ["xyz", s])


# ---- matcher level ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["auto", "list", "dense32", "block"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("k", [7, 33])
def test_matcher_frames_at_attained_thresholds(pf, gpu, monkeypatch, variant, mode, k):
    """TFIDF(min_similarity=v, top_n=k) at attained v, with the variant it picks itself or a forced one: the frame equals
    the assembled oracle lists."""
    polyfuzz_b200, engine = pf
    if variant != "auto":
        _force_variant(monkeypatch, engine, variant)
    run = gpu.runs[mode][1]
    for ms in (run, math.nextafter(run, -math.inf), 1.0, math.nextafter(1.0, 0.0)):
        m = polyfuzz_b200.TFIDF(min_similarity=ms, top_n=k)
        df = m.match(gpu.case.frm, gpu.case.to) if mode == "two" else m.match(gpu.case.to)
        oi, ov = gpu.oracle(mode, ms)
        ref = oracle_assemble(gpu.case.from_list(mode), gpu.case.to, oi[:, :k], ov[:, :k])
        _frame_eq(df, ref)
