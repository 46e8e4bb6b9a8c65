"""K7, single linkage on the device (polyfuzz_b200.single_linkage), against the reference's single_linkage byte-compiled
into oracle/_ref by build(): the three dicts must be equal in content and iteration order.  Also the unmodified
PolyFuzz.group with install_linkage(), and the refusal of kept rows whose keys are not str."""
import json
import os

import numpy as np
import pandas as pd
import pytest

import linkage_model as lm

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
REF = os.path.join(ROOT, "oracle", "_ref")
FROM = ["apple", "apples", "appl", "recal", "house", "similarity"]
TO = ["apple", "apples", "mouse"]


@pytest.fixture(scope="module")
def ref():
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference orchestrator) was not built")
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    from oracle import ref_shim
    ref_shim.REFERENCE_ROOT = REF
    ref_shim.install()
    import polyfuzz.linkage
    return polyfuzz.linkage.single_linkage


def _device(frame, thr):
    from polyfuzz_b200 import single_linkage
    return single_linkage(frame, thr)


def _check(ref, frame, thr):
    want = ref(frame, thr)
    got = _device(frame, thr)
    assert lm.as_lists(got) == lm.as_lists(want)
    assert all(type(v) is int for v in got[1].values())


def test_random_and_group_shaped_frames(ref):
    rng = np.random.default_rng(20261017)
    for i in range(300):
        n = int(rng.integers(1, 400))
        if i % 2:
            frame = lm.random_frame(rng, n, pool=int(rng.integers(1, 2 * n + 2)), self_rate=float(rng.choice([0.0, 0.2, 0.6])))
        else:
            frame = lm.random_frame(rng, n, pool=n, unique_from=True, self_rate=0.3)
        _check(ref, frame, float(rng.choice(lm.SCORES)))


def test_large_random_frames(ref):
    rng = np.random.default_rng(5)
    for n, pool, uf in ((100_000, 100_000, True), (200_000, 50_000, False)):
        frame = lm.random_frame(rng, n, pool=pool, unique_from=uf, self_rate=0.05)
        _check(ref, frame, 0.75)


def test_hubs_retarget_empty_and_strict_threshold(ref):
    rng = np.random.default_rng(3)
    for hubs in (1, 3):
        _check(ref, lm.hub_frame(rng, 20_000, hubs), 0.5)
    mixed = pd.concat([lm.hub_frame(rng, 3000, 1), lm.random_frame(rng, 500, 600)], ignore_index=True)
    _check(ref, mixed.sample(frac=1.0, random_state=1).reset_index(drop=True), 0.6)
    _check(ref, lm.retarget_frame(), 0.5)
    frame = lm.random_frame(rng, 300, 200, self_rate=0.1)
    for thr in (1.0, 2.0):
        assert lm.as_lists(_device(frame, thr)) == [[], [], []]
    assert lm.as_lists(_device(frame.iloc[:0], 0.5)) == [[], [], []]
    frame["Similarity"] = np.where(np.arange(300) % 2, 0.75, 0.9)
    frame.loc[::7, "Similarity"] = np.nan
    for thr in (0.75, np.nextafter(0.75, 0.0), 0.9):
        _check(ref, frame, thr)


@pytest.mark.parametrize("reverse", [False, True])
def test_long_chain_runs_the_finish_kernel(ref, reverse):
    # s0 -> s1 -> ...: each create waits for the row before it, so far more than the enqueued rounds are needed
    _check(ref, lm.chain_frame(200_001, reverse=reverse), 0.5)


def test_device_threshold_equals_host_filter():
    from polyfuzz_b200.linkage import linkage_arrays
    rng = np.random.default_rng(9)
    n, keys = 50_000, 20_000
    F, T = rng.integers(0, keys, n), rng.integers(0, keys, n)
    sim = lm.SCORES[rng.integers(0, len(lm.SCORES), n)].copy()
    sim[::11] = np.nan
    for thr in (0.75, 0.0, 1.0):
        kept = sim > thr
        a = linkage_arrays(F, T, keys, similarity=sim, min_similarity=thr)
        b = linkage_arrays(F[kept], T[kept], keys)
        assert all(np.array_equal(x, y) for x, y in zip(a[:4], b[:4])) and a[4] == b[4]
        val, rank, rep, _ = lm.linkage_ids(F[kept], T[kept], keys)
        assert np.array_equal(a[0], val) and np.array_equal(a[1], rank) and np.array_equal(a[2], rep)


@pytest.mark.parametrize("lo", [0, 60_000])
def test_company_name_self_matches(ref, lo):
    from polyfuzz_b200 import TFIDF
    names = json.load(open(os.path.join(ROOT, "tests", "golden", "data", "company_names.json")))[lo:lo + 30_000]
    frame = TFIDF(n_gram_range=(3, 3), min_similarity=0).match(names)
    for thr in (0.5, 0.75, 0.9):
        _check(ref, frame, thr)
        assert 1 <= lm.rounds_of(frame, thr) <= 12


def test_null_or_non_str_kept_key_is_refused(ref):
    frame = pd.DataFrame({"From": ["a", "b", "c"], "To": ["b", None, "a"], "Similarity": [0.9, 0.0, 0.9]})
    _check(ref, frame, 0.5)                                     # the null row is not kept
    with pytest.raises(ValueError, match="str"):
        _device(frame, -1.0)
    frame = pd.DataFrame({"From": ["a", 3, "c"], "To": ["b", "a", "a"], "Similarity": [0.9, 0.9, 0.9]})
    with pytest.raises(ValueError, match="str"):
        _device(frame, 0.5)


@pytest.fixture()
def polyfuzz_pkg(ref):
    import polyfuzz
    import polyfuzz.polyfuzz as pp
    return polyfuzz, pp


def _group(PolyFuzz, TFIDF, frm, to, group_all_strings):
    model = PolyFuzz(TFIDF(min_similarity=0)).match(frm, to)
    model.group(model=TFIDF(n_gram_range=(3, 3), min_similarity=0.75), link_min_similarity=0.75, group_all_strings=group_all_strings)
    return model.get_matches(), model.get_clusters(), model.get_cluster_mappings()


@pytest.mark.parametrize("group_all_strings", [False, True])
def test_group_with_install_linkage(polyfuzz_pkg, monkeypatch, group_all_strings):
    polyfuzz, pp = polyfuzz_pkg
    import polyfuzz.linkage as pl
    import polyfuzz_b200
    from polyfuzz_b200 import TFIDF
    names = json.load(open(os.path.join(ROOT, "tests", "golden", "data", "company_names.json")))
    frm, to = names[40_000:44_000], names[42_000:48_000]
    cases = [(FROM, TO), (FROM, FROM), (frm, to), (frm, frm)]
    want = [_group(polyfuzz.PolyFuzz, TFIDF, a, b, group_all_strings) for a, b in cases]
    monkeypatch.setattr(pp, "single_linkage", pp.single_linkage)
    monkeypatch.setattr(pl, "single_linkage", pl.single_linkage)
    polyfuzz_b200.install_linkage()
    assert pp.single_linkage is polyfuzz_b200.single_linkage and pl.single_linkage is polyfuzz_b200.single_linkage
    for (a, b), (wm, wc, wmap) in zip(cases, want):
        gm, gc, gmap = _group(polyfuzz.PolyFuzz, TFIDF, a, b, group_all_strings)
        pd.testing.assert_frame_equal(gm, wm)
        assert list(gc.items()) == list(wc.items()) and list(gmap.items()) == list(wmap.items())
    if not group_all_strings:
        assert _group(polyfuzz.PolyFuzz, TFIDF, FROM, TO, False)[1] == {1: ["apples", "apple"]}   # tests/test_polyfuzz.py:85-86
    else:
        assert _group(polyfuzz.PolyFuzz, TFIDF, FROM, FROM, True)[1] == {1: ["apples", "apple", "appl"]}
