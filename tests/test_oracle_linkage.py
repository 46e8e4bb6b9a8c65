"""The round model of single linkage (tests/linkage_model.py, the rule K7 implements) against the reference's own
single_linkage, with the iteration order of all three dicts compared.  No GPU: this pins the algorithm by itself."""
import numpy as np
import pandas as pd
import pytest

import linkage_model as lm
from oracle import ref_shim

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="the reference is not present")


@pytest.fixture(scope="module")
def ref_linkage():
    ref_shim.install()
    from polyfuzz.linkage import single_linkage
    return single_linkage


def _check(ref_linkage, frame, thr):
    want = lm.as_lists(ref_linkage(frame, thr))
    got = lm.as_lists(lm.single_linkage(frame, thr))
    assert got == want


def test_random_frames_with_repeated_from_and_self_rows(ref_linkage):
    rng = np.random.default_rng(20261017)
    for _ in range(400):
        n = int(rng.integers(1, 60))
        frame = lm.random_frame(rng, n, pool=int(rng.integers(1, 2 * n + 2)), self_rate=float(rng.choice([0.0, 0.2, 0.6])))
        _check(ref_linkage, frame, float(rng.choice(lm.SCORES)))


def test_group_shaped_frames(ref_linkage):
    rng = np.random.default_rng(7)
    for _ in range(300):
        n = int(rng.integers(1, 200))
        frame = lm.random_frame(rng, n, pool=n, unique_from=True, self_rate=0.3)
        _check(ref_linkage, frame, float(rng.choice([0.0, 0.5, 0.75, 0.9])))


@pytest.mark.parametrize("reverse", [False, True])
def test_chains(ref_linkage, reverse):
    frame = lm.chain_frame(300, reverse=reverse)
    _check(ref_linkage, frame, 0.5)
    if not reverse:
        assert lm.rounds_of(frame, 0.5) >= 149                     # alternating create / skip: one round per create


def test_hubs(ref_linkage):
    rng = np.random.default_rng(3)
    for hubs in (1, 3):
        frame = lm.hub_frame(rng, 5000, hubs)
        _check(ref_linkage, frame, 0.5)
    # a hub shuffled among random rows, so that creates, inherits and skips on the hub key interleave
    frame = pd.concat([lm.hub_frame(rng, 3000, 1), lm.random_frame(rng, 500, 600)], ignore_index=True)
    _check(ref_linkage, frame.sample(frac=1.0, random_state=1).reset_index(drop=True), 0.6)


def test_r0_keys_retargeted(ref_linkage):
    frame = lm.retarget_frame()
    _check(ref_linkage, frame, 0.5)
    assert 0 not in lm.single_linkage(frame, 0.5)[1].values()      # both of r0's keys end in later clusters


def test_empty_kept_set(ref_linkage):
    rng = np.random.default_rng(1)
    frame = lm.random_frame(rng, 20, 10)
    for thr in (1.0, 2.0):
        assert lm.as_lists(ref_linkage(frame, thr)) == [[], [], []] == lm.as_lists(lm.single_linkage(frame, thr))
    empty = frame.iloc[:0]
    assert lm.as_lists(ref_linkage(empty, 0.5)) == lm.as_lists(lm.single_linkage(empty, 0.5))


def test_threshold_equal_to_a_score_is_strict(ref_linkage):
    rng = np.random.default_rng(11)
    frame = lm.random_frame(rng, 200, 150, unique_from=False, self_rate=0.1)
    frame["Similarity"] = np.where(np.arange(200) % 2, 0.75, 0.9)
    for thr in (0.75, np.nextafter(0.75, 0.0), 0.9):
        _check(ref_linkage, frame, thr)
    nan = frame.copy()
    nan.loc[::3, "Similarity"] = np.nan                           # NaN fails the test, as in pandas
    _check(ref_linkage, nan, 0.5)


def test_readme_group_frame(ref_linkage):
    # shaped like the self-match group() links for the README lists: r0's cluster id 0 is falsy, so the cluster is 1
    frame = pd.DataFrame({"From": ["apple", "apples", "mouse"], "To": ["apples", "apple", None], "Similarity": [0.783, 0.783, 0.0]})
    assert lm.single_linkage(frame, 0.75)[0] == {1: ["apples", "apple"]} == ref_linkage(frame, 0.75)[0]
