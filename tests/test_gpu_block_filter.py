"""The block kernel's filter (spcos_blk3_kernel, DESIGN §4.1): a from-row's gate decides which cells go to exact re-scoring.
The gate only filters, so results must stay bit-identical to the oracle wherever the gate's rules change course: self-match
and two lists, a cutoff above most scores, rows with fewer than K neighbours or only very common trigrams, exact ties at the
K-th score, tiles and tile splits, a shard of the to-side, both accumulator widths and every block size.  On the company
slice the number of candidates the GPU filter queues (gcnt) must agree with the CPU model of tools/k2_cand_count.py."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import native as onative

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


@pytest.fixture(scope="module")
def engine():
    import polyfuzz_b200  # noqa: F401  (builds / loads the library)
    from polyfuzz_b200 import engine
    return engine


@pytest.fixture(scope="module")
def names():
    data = json.load(open(os.path.join(ROOT, "tests", "golden", "data", "company_names.json")))
    # real names, plus rows the seed pass cannot seed: only heavy trigrams (no light terms), strings with fewer than K
    # neighbours, an empty row, and groups of exact duplicates (ties at the K-th score)
    odd = ["inc", "llc", "inc llc", "corp inc", "", "qqxzj vvwk", "zyxw", "ab"]
    dups = ["acme holdings inc"] * 25 + ["acme holding inc"] * 9 + ["global trading company ltd"] * 14
    return list(data[:5000]) + odd + dups


def _set_shape(monkeypatch, engine, acc_bits, rows):
    monkeypatch.setattr(engine, "BLOCK_ACC_BITS", acc_bits)
    monkeypatch.setattr(engine, "BLOCK_ROWS", rows)


def _check(engine, csr_from, csr_to, k, ms, self_match, tile, splits, to_index_base=0, oracle=None):
    ix = engine.SparseIndex(csr_to, tile=tile, variant="block")
    idx, val = engine.spcos_topk(csr_from, ix, k, ms, self_match=self_match, n_splits=splits, to_index_base=to_index_base,
                                 variant="block")
    assert int(ix._block_err.item()) == 0
    if oracle is None:
        oracle = onative.spdot_topn(csr_from.to_scipy(), csr_to.to_scipy(), k, ms, self_match=self_match,
                                    to_index_base=to_index_base, n_threads=8)
    oi, ov = oracle
    assert (idx.cpu().numpy() == oi).all()
    assert (val.cpu().numpy() == ov).all()


@pytest.mark.parametrize("acc_bits,rows", [(16, 8), (32, 8), (16, 4), (32, 4), (16, 16), (32, 16)])
def test_self_match_tiles_and_splits(engine, monkeypatch, names, acc_bits, rows):
    _set_shape(monkeypatch, engine, acc_bits, rows)
    v = engine.NgramTfidf((3, 3), True, True)
    (r,) = v.fit_rows([names]); csr = v.emit(r)
    a = csr.to_scipy()
    oracle = onative.spdot_topn(a, a, 10, 0.0, self_match=True, n_threads=8)
    for tile, splits in ((128, 1), (1024, 1), (4096, 1), (1024, 3), (256, 2)):
        if acc_bits == 32 and tile > 2048:
            tile = 2048                                      # (32-bit accumulators: half the tile in the same shared memory)
        _check(engine, csr, csr, 10, 0.0, True, tile, splits, oracle=oracle)


@pytest.mark.parametrize("acc_bits", [16, 32])
@pytest.mark.parametrize("ms", [0.0, 0.6])
@pytest.mark.parametrize("k", [10, 3, 32])
def test_two_lists_and_cutoff(engine, monkeypatch, names, acc_bits, ms, k):
    """A cutoff of 0.6 lies above the K-th score of most rows: the gate starts from the cutoff, not from the sums."""
    _set_shape(monkeypatch, engine, acc_bits, 8)
    to, frm = names[:3500], names[3000:]
    v = engine.NgramTfidf((3, 3), True, True)
    rows_to, rows_from = v.fit_rows([to, frm])
    csr_to, csr_from = v.emit(rows_to), v.emit(rows_from)
    _check(engine, csr_from, csr_to, k, ms, False, 1024, 1)
    _check(engine, csr_from, csr_to, k, ms, False, 256, 3)


@pytest.mark.parametrize("acc_bits", [16, 32])
def test_shard_of_the_to_side(engine, monkeypatch, names, acc_bits):
    """A self-match against one shard of the to-side (non-zero to_index_base): the diagonal is only in that shard."""
    _set_shape(monkeypatch, engine, acc_bits, 8)
    v = engine.NgramTfidf((3, 3), True, True)
    (r,) = v.fit_rows([names]); csr = v.emit(r)
    a = csr.to_scipy()
    lo, hi = 1700, 3900
    shard = v.transform(names[lo:hi])
    oracle = onative.spdot_topn(a, shard.to_scipy(), 10, 0.0, self_match=True, to_index_base=lo, n_threads=8)
    _check(engine, csr, shard, 10, 0.0, True, 1024, 1, to_index_base=lo, oracle=oracle)
    _check(engine, csr, shard, 10, 0.0, True, 512, 2, to_index_base=lo, oracle=oracle)


def _gcnt_mean(engine, csr, tile):
    """Mean candidates per from-row the block kernel left for exact re-scoring (its gcnt array), read from its workspace."""
    from polyfuzz_b200 import _lib
    orig_ws = engine._ws
    kept = []
    engine._ws = lambda nbytes: kept.append(orig_ws(nbytes)) or kept[-1]
    try:
        ix = engine.SparseIndex(csr, tile=tile, variant="block")
        kept.clear()
        engine.spcos_topk(csr, ix, 10, 0.0, self_match=True, n_splits=1, variant="block")
        torch.cuda.synchronize()
    finally:
        engine._ws = orig_ws
    n = csr.n_rows
    off = _lib.load().pfz_spcos_block_gcnt_offset(n, int(csr.indices.numel()), ix.n_vocab, 1)
    return float(kept[0][off:off + 4 * n].view(torch.int32).double().mean())


def test_candidate_count_matches_the_cpu_model(engine, monkeypatch):
    """Company slice (3 000 names), tile 1 024, top-10: the CPU model (tools/k2_cand_count.py --names
    tests/golden/company_slice_names.json --rows 3000 --tile 1024) counts 31.0 candidates per row, and 10.5 with a gate
    that starts at the row's true K-th score.  The GPU sums are fixed point and its groups are visited in another order,
    so the count only has to agree within a margin."""
    _set_shape(monkeypatch, engine, 16, 8)
    sl = json.load(open(os.path.join(ROOT, "tests", "golden", "company_slice_names.json")))["names"]
    v = engine.NgramTfidf((3, 3), True, True)
    (r,) = v.fit_rows([sl]); csr = v.emit(r)
    mean = _gcnt_mean(engine, csr, 1024)
    assert 0.7 * 31.0 < mean < 1.3 * 31.0, mean
