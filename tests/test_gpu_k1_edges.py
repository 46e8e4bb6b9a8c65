"""K1 (the n-gram TF-IDF vectoriser) at the places where it changes path, bit-exact against the unmodified reference
(inputs from tests/k1_cases.py, outputs in tests/golden/k1_edges.npz, made by tests/golden/make_golden.py --k1-edges):
  - rows of 255 / 256 / 257 n-gram slots (ngram_rows_warp_kernel -> ngram_rows_long_kernel above WARP_ROW_SLOTS) and of
    8 191 / 8 192 slots (the long kernel's key arena is full at MAX_ROW_SLOTS), mixed with short and empty rows;
  - a code space of exactly DENSE_CODE_SPACE_MAX = 2^24 (direct-addressed df table) and one just above it (gather + sort);
  - n-gram codes >= 2^63, which sit in int64 tensors.
Each test also asserts which path it reached, so that a changed threshold cannot turn it into an ordinary test."""
import pickle

import numpy as np
import pytest

import k1_cases

pytestmark = pytest.mark.gpu

DENSE = {"slots33_clean": True, "slots33_raw": True, "slots13_clean": True, "slots36_raw": False, "slots18_raw": False,
         "space255_raw33": True, "space256_raw33": False, "codes64_raw18": False, "codes64_raw88": False}


@pytest.fixture(scope="module")
def engine():
    from polyfuzz_b200 import engine
    return engine


@pytest.fixture(scope="module")
def cases(golden_dir):
    return k1_cases.load(golden_dir)


def _csr_eq(dev_csr, g, part):
    m = dev_csr.to_scipy()
    assert m.shape == tuple(g[part + "_shape"])
    np.testing.assert_array_equal(m.indptr, g[part + "_indptr"])
    np.testing.assert_array_equal(m.indices, g[part + "_indices"])
    assert m.data.view(np.uint64).tolist() == g[part + "_data"].view(np.uint64).tolist()      # fp64 bits


def _slots(strings, lo, hi):
    from polyfuzz_b200.strings import ngram_slot_bounds
    off = np.zeros(len(strings) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(s) for s in strings])
    return ngram_slot_bounds(off, lo, hi)[0]


def _check_fitted(v, c, rows_to, rows_from):
    g = c["g"]
    assert v.vocabulary() == c["vocabulary"]
    assert v.idf.view(np.uint64).tolist() == g["idf"].view(np.uint64).tolist()
    _csr_eq(v.emit(rows_to), g, "to")
    _csr_eq(v.emit(rows_from), g, "from")
    _csr_eq(v.transform(c["new"]), g, "new")


@pytest.mark.parametrize("name", k1_cases.NAMES)
def test_k1_edges_match_reference(engine, cases, name):
    c = cases[name]
    g = c["g"]
    lo, hi = c["ngram_range"]
    # path: rows above WARP_ROW_SLOTS run the long kernel, and the fixture provably holds the targeted slot counts
    slots = np.concatenate([_slots(c["frm"], lo, hi), _slots(c["to"], lo, hi)])
    assert set(c["slots"]) <= set(slots.tolist())
    assert slots.max() <= engine.MAX_ROW_SLOTS
    staged = [engine.stage_strings(lst, lo, hi) for lst in (c["to"], c["frm"])]
    for S, lst in zip(staged, (c["to"], c["frm"])):
        assert S.n_long == int((_slots(lst, lo, hi) > engine.WARP_ROW_SLOTS).sum())
    assert sum(S.n_long for S in staged) > 0
    if c["slots"]:
        assert any(s > engine.WARP_ROW_SLOTS for s in c["slots"]) and any(s <= engine.WARP_ROW_SLOTS for s in c["slots"])

    v = engine.NgramTfidf((lo, hi), c["clean"], c["remove_space"])
    rows_to, rows_from = v.fit_staged(staged)
    # path: direct-addressed df table (and rank table) iff the code space is at most 2^24
    assert (v.code_space() <= engine.DENSE_CODE_SPACE_MAX) == DENSE[name]
    assert (v._d_rank is not None) == DENSE[name]
    if name.startswith("space"):
        assert v.base - 1 == (255 if name == "space255_raw33" else 256)
        assert v.code_space() == (1 << 24 if name == "space255_raw33" else 257 ** 3)
        assert (v.alphabet > 0xFF).sum() == len(v.alphabet) - 1                # every symbol but the space is past Latin-1
    if name.startswith("codes64"):
        assert v.base - 1 == 254 and 2 ** 63 < v.code_space() < 2 ** 64
        assert (v.vocab_keys >= np.uint64(1 << 63)).sum() > 100             # codes >= 2^63 are in the vocabulary
    _check_fitted(v, c, rows_to, rows_from)

    # pickle round trip: device state is rebuilt from the host copies (the rank table only for a dense code space)
    v2 = pickle.loads(pickle.dumps(v))
    assert v2._d_vocab is None
    _csr_eq(v2.transform(c["new"]), g, "new")
    assert (v2._d_rank is not None) == DENSE[name]
    _csr_eq(v2.transform(c["frm"]), g, "from")
    _csr_eq(v2.transform(c["to"]), g, "to")
    assert v2.vocabulary() == c["vocabulary"]


def test_k1_refuses_rows_above_max_row_slots(engine):
    """8 193 slots: one more than the long kernel's key arena holds.  A documented refusal (DESIGN section 6)."""
    assert engine.MAX_ROW_SLOTS == 8192
    for lo, hi, L in ((3, 3, 8195), (1, 3, 2732), (1, 8, 1028)):
        s = _slots(["x" * L], lo, hi)
        assert s[0] > engine.MAX_ROW_SLOTS and _slots(["x" * (L - 1)], lo, hi)[0] <= engine.MAX_ROW_SLOTS
        with pytest.raises(ValueError, match=rf"string 1 has {int(s[0])} n-gram slots; the vectoriser supports at most 8192"):
            engine.NgramTfidf((lo, hi), True, True).fit_rows([["ab", "x" * L, ""]])
    # the largest row that is accepted
    v = engine.NgramTfidf((3, 3), True, True)
    (rows,) = v.fit_rows([["a" * 8194, "ab"]])
    assert v.vocabulary() == ["aaa"]
    m = v.emit(rows).to_scipy()
    assert m.indptr.tolist() == [0, 1, 1] and m.data.tolist() == [1.0]


def test_k1_refuses_codes_beyond_64_bits(engine):
    """An alphabet of 255 symbols at (8,8): 256^8 = 2^64 codes do not fit 64 bits.  254 symbols do (codes64_raw88)."""
    alpha = k1_cases.alphabet(255)
    assert len(set(alpha)) == 255
    v = engine.NgramTfidf((8, 8), False, False)
    with pytest.raises(ValueError, match="alphabet of 255 symbols with 8-grams exceeds 64-bit n-gram codes"):
        v.fit_rows([[alpha, alpha[::-1]]])
    v = engine.NgramTfidf((8, 8), False, False)
    v.fit_rows([[alpha[1:], alpha[::-1][:-1]]])
    assert v.base - 1 == 254 and v.n_vocab > 0
