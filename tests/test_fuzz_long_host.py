"""Host logic of K3b's word classes (CPU only, the kernels stubbed): the class of each from-string length, the n_words each
pfz_fuzz_* call receives, the from-side limit of 1 024 code points and to-strings of any length."""
import numpy as np
import pytest
import torch

from polyfuzz_b200 import fuzzy


class _Calls:
    def __init__(self):
        self.fuzz = []

    def call(self, name, *args):
        if name.startswith("pfz_fuzz_"):
            self.fuzz.append((name, args[3], args[4]))        # (entry point, n_ids, n_words)


@pytest.fixture
def calls(monkeypatch):
    c = _Calls()
    monkeypatch.setattr(fuzzy, "_lib", c)
    monkeypatch.setattr(fuzzy, "_dev", lambda: torch.device("cpu"))
    monkeypatch.setattr(fuzzy, "_to_dev", lambda arr, dtype=None: (torch.from_numpy(np.ascontiguousarray(arr)) if dtype is None
                                                                  else torch.from_numpy(np.ascontiguousarray(arr)).view(dtype)))
    monkeypatch.setattr(fuzzy, "_blob_to_dev", lambda b: torch.from_numpy(np.ascontiguousarray(b).astype(np.int64)))
    monkeypatch.setattr(fuzzy, "_stream", lambda: None)
    monkeypatch.setattr(fuzzy, "_p", lambda t: None)
    return c


def test_word_class_map():
    lens = np.array([0, 1, 64, 65, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024])
    assert fuzzy.word_class(lens).tolist() == [1, 1, 1, 2, 2, 4, 4, 4, 8, 8, 8, 16, 16, 16]


@pytest.mark.parametrize("k", [None, 5])
def test_n_words_per_length(calls, k):
    frm = ["a" * n for n in (10, 100, 200, 256, 300, 512, 700, 1024)] + ["b c " * 100]    # last: 400 code points
    fuzzy._enqueue(frm, ["x" * 7000, "y"], "WRatio", 0.0, False, None, 0, 0, k)
    name = "pfz_fuzz_argbest" if k is None else "pfz_fuzz_topk"
    assert calls.fuzz == [(name, 1, 1), (name, 1, 2), (name, 2, 4), (name, 3, 8), (name, 2, 16)]


def test_from_limit_message_and_unbounded_to_side(calls):
    with pytest.raises(ValueError, match=r"from-string 1 has 1025 code points; the token / partial scorers support at most 1024"):
        fuzzy._enqueue(["a", "a" * 1025], ["b"], "WRatio", 0.0, False, None, 0, 0, None)
    assert calls.fuzz == []
    fuzzy._enqueue(["a b"], ["c " * 20000], "token_set_ratio", 0.0, False, None, 0, 0, 3)
    assert calls.fuzz == [("pfz_fuzz_topk", 1, 1)]
