"""CPU tests: pin the oracle against the golden vectors generated from the UNMODIFIED reference
(tests/golden/make_golden.py) and against the definition-level known answers of SURVEY.md 8c."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp

import k1_cases
from oracle import native, tfidf
from oracle.assemble import assemble, cosine_topk_dense

FROM = ["apple", "apples", "appl", "recal", "house", "similarity"]
TO = ["apple", "apples", "mouse"]
RANGES = [(1, 1), (1, 2), (1, 3), (2, 2), (2, 3), (3, 3), (3, 6)]


def _eq(m, g, prefix):
    m = m.tocsr(); m.sort_indices()
    np.testing.assert_array_equal(m.indptr, g[prefix + "_indptr"])
    np.testing.assert_array_equal(m.indices, g[prefix + "_indices"])
    np.testing.assert_array_equal(m.data, g[prefix + "_data"])


@pytest.mark.parametrize("lo,hi", RANGES)
@pytest.mark.parametrize("clean", [True, False])
@pytest.mark.parametrize("rs", [True, False])
def test_tfidf_oracles_match_reference_c1(golden_dir, lo, hi, clean, rs):
    g = np.load(os.path.join(golden_dir, "c1_tfidf.npz"))
    voc = json.load(open(os.path.join(golden_dir, "c1_vocab.json")))
    tag = f"r{lo}{hi}_c{int(clean)}_s{int(rs)}"
    f, t, vec = tfidf.fit_transform_sklearn(FROM, TO, (lo, hi), clean, rs)
    _eq(f, g, tag + "_two_from"); _eq(t, g, tag + "_two_to")
    o = tfidf.TfidfOracle((lo, hi), clean, rs).fit(TO + FROM)
    assert o.vocabulary == voc[tag + "_two"]
    np.testing.assert_array_equal(o.idf, g[tag + "_two_idf"])
    _eq(o.transform(FROM), g, tag + "_two_from"); _eq(o.transform(TO), g, tag + "_two_to")
    o2 = tfidf.TfidfOracle((lo, hi), clean, rs).fit(FROM)
    assert o2.vocabulary == voc[tag + "_self"]
    _eq(o2.transform(FROM), g, tag + "_self")


def test_c1_known_answers():
    """SURVEY.md 8c (1): vocabulary, idf and the 6x3 cosine matrix of the README lists."""
    o = tfidf.TfidfOracle().fit(TO + FROM)
    assert o.vocabulary == "app,ari,cal,eca,hou,ila,imi,ity,lar,les,mil,mou,ous,ple,ppl,rec,rit,sim,use".split(",")
    idf = dict(zip(o.vocabulary, o.idf))
    assert idf["app"] == 1.5108256237659907 and idf["ple"] == 1.6931471805599454
    assert idf["les"] == idf["ous"] == idf["use"] == 2.203972804325936 and idf["sim"] == 2.6094379124341005
    c = (o.transform(FROM) @ o.transform(TO).T).toarray()
    exp = np.array([[.9999999999999998, .7776515952538289, 0], [.7776515952538289, 1, 0], [.783751479433796, .60948558826424, 0],
                    [0, 0, 0], [0, 0, .5879265964444779], [0, 0, 0]])
    np.testing.assert_allclose(c, exp, rtol=0, atol=2e-16)


def test_clean_string_matches_reference_probe(golden_dir):
    g = json.load(open(os.path.join(golden_dir, "clean_survivors.json")))
    assert g["non_ascii_survivors"] == {"304": "aib", "8490": "akb"}
    for cp, r in g["ascii"].items():
        assert tfidf.clean_string("a" + chr(int(cp)) + "b") == r
    for cp, r in g["non_ascii_survivors"].items():
        assert tfidf.clean_string("a" + chr(int(cp)) + "b") == r
    for s, r in g["examples"].items():
        assert tfidf.clean_string(s) == r


@pytest.fixture(scope="module")
def company(golden_dir):
    g = np.load(os.path.join(golden_dir, "company_slice.npz"))
    names = json.load(open(os.path.join(golden_dir, "company_slice_names.json")))["names"]
    return g, names


def test_company_slice_vectoriser(company):
    g, names = company
    f, _, vec = tfidf.fit_transform_sklearn(names)
    _eq(f, g, "csr")
    o = tfidf.TfidfOracle().fit(names)
    np.testing.assert_array_equal(o.idf, g["idf"])
    _eq(o.transform(names), g, "csr")


def test_company_slice_topn_vs_unmodified_reference(company):
    """The C restatement of awesome_cossim_topn + canonical tie-break reproduces the reference's
    sklearn branch: every 3-dp score, and every index on rows without an exact tie in ranks 1..k+1."""
    g, names = company
    a = sp.csr_matrix((g["csr_data"], g["csr_indices"], g["csr_indptr"]), shape=tuple(g["csr_shape"]))
    idx, val = native.spdot_topn(a, a, 10, 0.0, self_match=True)
    np.testing.assert_array_equal(np.round(val, 3), g["ref_sims"])
    tf = g["ref_tiefree"]
    assert tf.sum() > 500
    nz = g["ref_topvals"] > 0
    assert ((idx == g["ref_idx"]) | ~nz)[tf].all()
    np.testing.assert_allclose(val[tf], g["ref_topvals"][tf], rtol=0, atol=1e-12)
    # threads do not change the result
    idx8, val8 = native.spdot_topn(a, a, 10, 0.0, self_match=True, n_threads=4)
    np.testing.assert_array_equal(idx, idx8); np.testing.assert_array_equal(val, val8)


def test_c1_frames_vs_reference(golden_dir):
    ref = json.load(open(os.path.join(golden_dir, "c1_match.json")))
    for top_n in (1, 2, 3):
        f, t, _ = tfidf.fit_transform_sklearn(FROM, TO)
        idx, val = native.spdot_topn(f, t, top_n, 0.0)
        df = assemble(FROM, TO, idx, val)
        exp = ref[f"two_top{top_n}_ms0.0"]
        for c in df.columns:
            assert [None if (isinstance(v, float) and np.isnan(v)) else v for v in df[c].tolist()] == exp[c]
        f, t, _ = tfidf.fit_transform_sklearn(FROM, None)
        idx, val = native.spdot_topn(f, t, top_n, 0.0, self_match=True)
        df = assemble(FROM, None, idx, val)
        exp = ref[f"self_top{top_n}_ms0.0"]
        for c in df.columns:
            assert [None if (isinstance(v, float) and np.isnan(v)) else v for v in df[c].tolist()] == exp[c]


def test_topk_merge_oracle():
    rng = np.random.default_rng(0)
    a = sp.random(200, 50, density=0.2, random_state=1, format="csr"); a.data = np.abs(a.data) + 0.1
    b = sp.random(300, 50, density=0.2, random_state=2, format="csr"); b.data = np.round(np.abs(b.data), 1) + 0.1
    full_i, full_v = native.spdot_topn(a, b, 7, 0.0)
    parts = [native.spdot_topn(a, b[lo:hi], 7, 0.0, to_index_base=lo) for lo, hi in ((0, 100), (100, 200), (200, 300))]
    mi, mv = native.topk_merge(np.stack([p[0] for p in parts]), np.stack([p[1] for p in parts]), 7)
    np.testing.assert_array_equal(mi, full_i); np.testing.assert_array_equal(mv, full_v)


# ---- edit distance: definition-level known answers (SURVEY.md 8c (4)) -------------------------------
def test_levenshtein_known_answers():
    d = native.editdist_matrix(FROM, TO, "lev")
    assert d.tolist() == [[0, 1, 4], [1, 0, 5], [1, 2, 5], [5, 6, 5], [4, 5, 1], [9, 9, 9]]


def test_ratio_known_answers():
    d = native.editdist_matrix(FROM, TO, "indel")
    la = np.array([len(s) for s in FROM])[:, None]; lb = np.array([len(s) for s in TO])[None, :]
    ratio = (1.0 - d / (la + lb)) * 100.0
    np.testing.assert_allclose(ratio[0], [100, 90.9090909090909, 20], rtol=1e-12)
    np.testing.assert_allclose(ratio[2], [88.8888888888889, 80, 0], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(ratio[4], [20, 18.181818181818176, 80], rtol=1e-9)
    bi, bs, bd = native.editdist_argbest(FROM, TO, "ratio")
    np.testing.assert_allclose(bs, [100, 100, 88.8888888888889, 40, 80, 13.333333333333329], rtol=1e-12)
    assert bs.mean() > 50                      # tests/models/test_distance.py:31 (normalize=False)
    # test_score_cutoff (tests/models/test_rapidfuzz.py:29-36): only exact matches survive 0.95
    bi, bs, _ = native.editdist_argbest(FROM, TO, "ratio", score_cutoff=95.0)
    assert bi.tolist() == [0, 1, -1, -1, -1, -1] and (bs / 100).mean() < 0.5


def test_myers_baseline_equals_dp():
    rng = np.random.default_rng(5)
    alpha = "abcdeé中"
    mk = lambda: "".join(alpha[i] for i in rng.integers(0, len(alpha), rng.integers(0, 70)))  # noqa: E731
    a = [mk() for _ in range(60)]; b = [mk() for _ in range(80)]
    i1, s1, d1 = native.editdist_argbest(a, b, "norm_lev")
    i2, s2, d2 = native.editdist_argbest(a, b, "norm_lev", myers=True, n_threads=2)
    np.testing.assert_array_equal(i1, i2); np.testing.assert_array_equal(d1, d2); np.testing.assert_array_equal(s1, s2)


def test_dense_fixture_vs_reference(golden_dir):
    g = np.load(os.path.join(golden_dir, "dense_c1.npz"))
    np.testing.assert_allclose(g["prod"][0], [1, .803842017962, .439652911433], atol=1e-9)
    for top_n in (1, 2, 3):
        idx, val = cosine_topk_dense(g["from_vec"], g["to_vec"], top_n, 0.0, normalize=True)
        np.testing.assert_array_equal(np.round(val, 3), g[f"sims_top{top_n}"])


@pytest.mark.parametrize("k,ms,self_match", [(1, 0.0, False), (5, 0.2, False), (4, 0.0, True), (50, 0.0, False)])
def test_two_oracle_statements_agree(k, ms, self_match):
    """Gustavson (C) vs the dense fp64 statement, on TF-IDF rows of real-looking strings: same indices under the
    canonical key; scores equal up to the different summation order of a dense dot product (<= 4 ulp)."""
    from polyfuzz_b200 import synth
    names = synth.company_names(700, seed=9) + ["dup co", "dup co", ""]
    to = names if self_match else synth.company_names(400, seed=10) + ["dup co"]
    f, t, _ = tfidf.fit_transform_sklearn(names, None if self_match else to)
    kk = min(k, t.shape[0])
    oi, ov = native.spdot_topn(f, t, kk, ms, self_match=self_match)
    di, dv = cosine_topk_dense(f.toarray(), t.toarray(), kk, ms, self_match=self_match)
    np.testing.assert_allclose(ov, dv, rtol=0, atol=1e-15)
    # rows whose consecutive scores differ by more than the summation noise must agree index for index
    gap = np.abs(np.diff(np.concatenate([dv, np.full((len(dv), 1), -1.0)], axis=1), axis=1))
    stable = (gap > 1e-12).all(axis=1) & (np.abs(dv - ms) > 1e-12).all(axis=1)
    assert stable.sum() > 50
    np.testing.assert_array_equal(oi[stable], di[stable])


def test_edit_distance_oracle_properties():
    rng = np.random.default_rng(11)
    alpha = "abcé中 "
    s = ["".join(alpha[i] for i in rng.integers(0, len(alpha), rng.integers(0, 25))) for _ in range(60)]
    d = native.editdist_matrix(s, s, "lev"); e = native.editdist_matrix(s, s, "indel")
    la = np.array([len(x) for x in s])
    assert (d == d.T).all() and (np.diag(d) == 0).all() and (e == e.T).all()
    assert (d >= np.abs(la[:, None] - la[None, :])).all() and (d <= np.maximum(la[:, None], la[None, :])).all()
    assert (e >= d).all() and (e <= 2 * d).all()                  # indel = lev with substitutions costed 2
    assert ((e - np.abs(la[:, None] - la[None, :])) % 2 == 0).all()
    # triangle inequality on a sample
    for a, b, c in rng.integers(0, len(s), (200, 3)):
        assert d[a, c] <= d[a, b] + d[b, c]


def test_fp32_filter_error_stays_below_half_the_margin():
    """The mixed-precision K2 variant (dense32) relies on |fp32 sum - exact score| < MARGIN/2 = 1e-5 for rows of at
    most 128 n-grams (polyfuzz_b200/engine.py: DENSE32_MAX_ROW_NNZ, csrc/pfz_spcos.cu: K2_MARGIN).  Emulate the fp32
    accumulation (weights rounded to fp32, running sum in fp32, worst of several term orders) on real TF-IDF rows,
    including rows close to the 128-term limit, and check the bound with room to spare."""
    from polyfuzz_b200 import synth
    rng = np.random.default_rng(4)
    words = synth.company_names(300, seed=12)
    long_rows = [" ".join(rng.choice(words, 6)) for _ in range(60)]          # ~100-128 distinct trigrams each
    names = synth.company_names(1500, seed=13) + long_rows
    a, _, _ = tfidf.fit_transform_sklearn(names)
    nnz = np.diff(a.indptr)
    assert nnz.max() > 100
    keep = np.nonzero(nnz <= 128)[0]
    dense = a[keep].toarray()
    d32 = dense.astype(np.float32)
    exact = dense @ dense.T
    worst = 0.0
    for trial in range(4):
        perm = rng.permutation(dense.shape[1])
        acc = np.zeros((len(keep), len(keep)), dtype=np.float32)
        blocks = np.array_split(perm, 64)                                    # 64 sequential fp32 partial additions
        for b in blocks:
            acc = (acc + d32[:, b] @ d32[:, b].T).astype(np.float32)
        worst = max(worst, float(np.abs(acc.astype(np.float64) - exact).max()))
    assert worst < 5e-6, worst


@pytest.mark.parametrize("tag,rng,clean", [("raw33", (3, 3), False), ("clean13", (1, 3), True), ("raw12", (1, 2), False)])
def test_titles_slice_vectoriser_matches_reference(golden_dir, tag, rng, clean):
    """Real movie titles (non-ASCII letters, punctuation, digits) from the reference's data/movie_titles.json:
    both oracle statements reproduce the unmodified reference's CSR and idf bit for bit, raw and clean mode."""
    g = np.load(os.path.join(golden_dir, "titles_slice.npz"))
    names = json.load(open(os.path.join(golden_dir, "titles_slice_names.json")))
    frm, to = names["from"], names["to"]
    assert any(ord(c) > 127 for s in frm + to for c in s)
    f, t, vec = tfidf.fit_transform_sklearn(frm, to, rng, clean, True)
    _eq(f, g, tag + "_from"); _eq(t, g, tag + "_to")
    o = tfidf.TfidfOracle(rng, clean, True).fit(list(to) + list(frm))
    np.testing.assert_array_equal(o.idf, g[tag + "_idf"])
    _eq(o.transform(frm), g, tag + "_from"); _eq(o.transform(to), g, tag + "_to")



@pytest.mark.parametrize("name", k1_cases.NAMES)
def test_k1_edges_oracles_match_reference(golden_dir, name):
    """Rows of 255..257 and 8 191..8 192 n-gram slots, code spaces of 2^24 and just above, codes >= 2^63 (tests/k1_cases.py):
    both oracle statements reproduce the unmodified reference's CSR, idf, vocabulary and transform bit for bit."""
    c = k1_cases.load(golden_dir)[name]
    g = {name + "_" + k: v for k, v in c["g"].items()}
    rng, clean, rs = tuple(c["ngram_range"]), c["clean"], c["remove_space"]
    f, t, vec = tfidf.fit_transform_sklearn(c["frm"], c["to"], rng, clean, rs)
    _eq(f, g, name + "_from"); _eq(t, g, name + "_to")
    _eq(vec.transform(c["new"]), g, name + "_new")
    o = tfidf.TfidfOracle(rng, clean, rs).fit(c["to"] + c["frm"])
    assert o.vocabulary == c["vocabulary"]
    np.testing.assert_array_equal(o.idf, g[name + "_idf"])
    _eq(o.transform(c["frm"]), g, name + "_from"); _eq(o.transform(c["to"]), g, name + "_to")
    _eq(o.transform(c["new"]), g, name + "_new")
