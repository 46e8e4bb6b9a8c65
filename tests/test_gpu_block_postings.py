"""The block kernel's postings (DESIGN §4.1).  In 16-bit mode pfz_index_pack_q15 packs each posting as exactly what the
update consumes: {byte offset of the accumulator word | byte-permute selector << 16, w15}.  The packing is checked bit for
bit against a numpy restatement of that layout.  The oversized-unit path (a unit with more work items than the kernel
stages, whose warps walk the term table and load the postings directly) is checked against the CPU oracle for both
accumulator widths."""
import numpy as np
import pytest
import torch

from oracle import native as onative

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    import polyfuzz_b200  # noqa: F401  (builds / loads the library)
    from polyfuzz_b200 import engine
    return engine


def _pack_q15(engine, idx, val, tile):
    from polyfuzz_b200 import _lib
    dev = torch.device("cuda")
    t_idx = torch.from_numpy(idx.astype(np.uint16).view(np.int16)).to(dev)
    t_val = torch.from_numpy(val).to(dev)
    nnz = torch.tensor([len(idx)], dtype=torch.int32, device=dev)
    out = torch.full((len(idx), 2), -1, dtype=torch.int32, device=dev)
    _lib.call("pfz_index_pack_q15", engine._p(t_idx), engine._p(t_val), engine._p(nnz), tile, engine._p(out), engine._stream())
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint32)


def _q15_layout(idx, val, tile):
    """x: byte offset of word j mod tile/2 | selector << 16 (0x4432: lower half-word, 0x3244: upper, j >= tile/2);
    y: w15 = max(1, round(w * 2^15)), ties to even"""
    j = idx.astype(np.uint32)
    half = np.uint32(tile // 2)
    hi = j >= half
    word = np.where(hi, j - half, j)
    x = (word << 2) | (np.where(hi, 0x3244, 0x4432).astype(np.uint32) << 16)
    w15 = np.maximum(1, np.rint(val * 32768.0)).astype(np.uint32)
    return np.stack([x, w15], axis=1)


@pytest.mark.parametrize("tile", [256, 4096])
def test_pack_q15_layout(engine, tile):
    rows = np.array([0, tile // 2 - 1, tile // 2, tile - 1], dtype=np.int64)
    weights = np.array([
        1.0,                                  # w15 = 32 768
        1e-7, 2.0 ** -17,                     # round to 0 and clamp to 1
        1 / 65536, 3 / 65536, 5 / 65536, 2001 / 65536, 32767 / 65536,   # w * 2^15 exactly .5: ties to even
        0.5, 0.123456789, 0.999999, 0.7071067811865476,
    ])
    idx = np.repeat(rows, len(weights))
    val = np.tile(weights, len(rows))
    rng = np.random.default_rng(7)
    idx = np.concatenate([idx, rng.integers(0, tile, 4000)])
    val = np.concatenate([val, rng.random(4000)])
    got = _pack_q15(engine, idx, val, tile)
    assert np.array_equal(got, _q15_layout(idx, val, tile))
    assert got[0, 1] == 32768
    assert list(got[len(weights) * np.arange(4), 0]) == [0x4432 << 16, (0x4432 << 16) | (4 * (tile // 2 - 1)),
                                                         0x3244 << 16, (0x3244 << 16) | (4 * (tile // 2 - 1))]


@pytest.mark.parametrize("tile", [128, 8448, 1000])
def test_pack_q15_refuses_tiles_outside_its_range(engine, tile):
    with pytest.raises(RuntimeError, match="pfz_index_pack_q15"):
        _pack_q15(engine, np.zeros(4, dtype=np.int64), np.full(4, 0.5), tile)


@pytest.mark.parametrize("acc_bits", [16, 32])
def test_oversized_unit(engine, monkeypatch, acc_bits):
    """From-rows that all hold the same 24 trigrams, which every to-row holds too: a (block, tile) unit is 24 terms x 1 024
    postings = 768 work items, more than the 8 x 64 the kernel stages, so its warps walk the term table directly."""
    monkeypatch.setattr(engine, "BLOCK_ACC_BITS", acc_bits)
    monkeypatch.setattr(engine, "BLOCK_ROWS", 8)
    base = "abcdefghijklmnopqrstuvwxyz"
    rng = np.random.default_rng(3)
    letters = np.array(list("abcdefghijklmnopqrstuvwxyz0123456789"))
    to = [base + " " + "".join(rng.choice(letters, int(rng.integers(1, 12)))) for _ in range(2300)]
    frm = [base] * 8 + to[:24]
    v = engine.NgramTfidf((3, 3), True, True)
    rows_to, rows_from = v.fit_rows([to, frm])
    csr_to, csr_from = v.emit(rows_to), v.emit(rows_from)
    assert int(np.diff(csr_from.to_scipy().indptr)[0]) == 24
    oi, ov = onative.spdot_topn(csr_from.to_scipy(), csr_to.to_scipy(), 10, 0.0, n_threads=8)
    ix = engine.SparseIndex(csr_to, tile=1024, variant="block")
    assert ix.tile == 1024 and ix.acc_bits == acc_bits
    idx, val = engine.spcos_topk(csr_from, ix, 10, 0.0, n_splits=1, variant="block")
    assert int(ix._block_err.item()) == 0
    assert (idx.cpu().numpy() == oi).all()
    assert (val.cpu().numpy() == ov).all()
