"""The TF-IDF driver (distributed.tfidf_topk_sharded) on one GPU, fitting on the to-list only (fit_on_from=False, what
TFIDF.match(from_block=...) runs) with an n-gram code space above 2^24: the from-list must add nothing to the vocabulary
or the df, and the result must equal a fit on the to-list alone, bit for bit."""
import numpy as np
import pytest

from oracle import native as onative
from oracle import tfidf as otfidf

pytestmark = pytest.mark.gpu

_SYMBOL = {" ": 1, **{chr(48 + i): 2 + i for i in range(10)}, **{chr(97 + i): 12 + i for i in range(26)}}


def _keys(vocabulary, hi):
    """The vectoriser's codes of cleaned n-grams: symbols in base 38, most significant first, shorter n-grams zero-padded
    at the end (so ascending codes are alphabetical order)."""
    out = []
    for g in vocabulary:
        key = 0
        for i in range(hi):
            key = key * 38 + (_SYMBOL[g[i]] if i < len(g) else 0)
        out.append(key)
    return np.array(out, dtype=np.uint64)


def _csr_eq(dev_csr, want):
    got = dev_csr.to_scipy()
    assert got.shape == want.shape
    np.testing.assert_array_equal(got.indptr, want.indptr)
    np.testing.assert_array_equal(got.indices, want.indices)
    np.testing.assert_array_equal(got.data.view(np.int64), want.data.view(np.int64))


def test_fit_on_to_list_only_with_a_large_code_space():
    from polyfuzz_b200 import engine, synth
    from polyfuzz_b200.distributed import tfidf_topk_sharded
    rng, k = (3, 5), 10
    assert 38 ** rng[1] > engine.DENSE_CODE_SPACE_MAX
    to = synth.company_names(3000, seed=21)
    frm = synth.company_names(500, seed=22) + to[:50] + ["zyxw vutsr", "qqqq jjjj 9876", "xkcd 0042"]
    o = otfidf.TfidfOracle(rng).fit(to)
    assert set(otfidf.TfidfOracle(rng).fit(to + frm).vocabulary) > set(o.vocabulary)   # the from-list brings n-grams of its own

    vec = engine.NgramTfidf(rng, True, True)
    idx, val, csr_to, index = tfidf_topk_sharded(vec, vec.stage(frm), vec.stage(to), 0, k, 0.0, False, fit_on_from=False)
    np.testing.assert_array_equal(vec.vocab_keys, _keys(o.vocabulary, rng[1]))
    np.testing.assert_array_equal(vec.df, o.df)
    np.testing.assert_array_equal(vec.idf.view(np.int64), o.idf.view(np.int64))
    assert vec.n_fit_docs == len(to)
    want_to, want_from = o.transform(to), o.transform(frm)
    _csr_eq(csr_to, want_to)
    _csr_eq(vec.transform(frm), want_from)
    oi, ov = onative.spdot_topn(want_from, want_to, k, 0.0, n_threads=8)
    np.testing.assert_array_equal(idx.cpu().numpy(), oi)
    np.testing.assert_array_equal(val.cpu().numpy().view(np.int64), ov.view(np.int64))
