"""K3b's token tables built on the device (pfz_tok_*) against the host oracle (tests/tok_oracle.py), array by array with ==,
and the kept to-side of RapidFuzz / EditDistance: a re_train=False call gives the frame a fresh matcher's call gives."""
import os
import pickle
import random
import sys

import numpy as np
import pandas as pd
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tok_oracle  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
REF = os.path.join(ROOT, "oracle", "_ref")
SPACES = [0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x1C, 0x1D, 0x1E, 0x1F, 0x20, 0x85, 0xA0, 0x1680] + list(range(0x2000, 0x200B)) + \
         [0x2028, 0x2029, 0x202F, 0x205F, 0x3000]


def _device_tables(from_list, to_list=None):
    """The device buffers of one call, trimmed to their filled lengths, in the oracle's layout."""
    from polyfuzz_b200 import fuzzy
    same = to_list is None
    F = fuzzy.TokSide(from_list)
    T = F if same else fuzzy.TokSide(to_list)
    f_ids, f_sig, t_ids, t_sig, tok_blob, tok_off = fuzzy._call_ids(F, T, same)
    torch.cuda.synchronize()

    def side(S, ids, sig):
        def blob(b, o):
            o = o.cpu().numpy()
            return b.cpu().numpy()[:o[-1]], o
        ptr = S.d_tok_ptr.cpu().numpy()
        return {"s": blob(S.d_blob, S.d_off), "S": blob(*S.d_S), "U": blob(*S.d_U), "tok_ptr": ptr,
                "tok_ids": ids.cpu().numpy()[:ptr[-1]], "sig": sig.cpu().numpy().view(np.uint64)[:S.n],
                "n_all": S.d_n_all.cpu().numpy()[:S.n]}

    n_u = F.n_vocab if same else int(T.n_vocab + F.n_vocab)   # an upper bound; trimmed by the offsets below
    off = tok_off.cpu().numpy()[:n_u + 1]
    return side(F, f_ids, f_sig), side(T, t_ids, t_sig), tok_blob.cpu().numpy(), off


def _check(from_list, to_list=None):
    Fd, Td, vblob, voff = _device_tables(from_list, to_list)
    Fo, To, vocab = tok_oracle.tables(from_list, to_list)
    for got, exp in ((Fd, Fo), (Td, To)):
        for key in ("s", "S", "U"):
            assert np.array_equal(got[key][1], exp[key][1]), key
            assert np.array_equal(got[key][0].astype(np.int64), exp[key][0].astype(np.int64)), key
        for key in ("tok_ptr", "tok_ids", "sig", "n_all"):
            assert got[key].dtype == exp[key].dtype and np.array_equal(got[key], exp[key]), key
    eb, eo = tok_oracle._cps(vocab)
    assert np.array_equal(voff[:len(vocab) + 1], eo)
    assert np.all(voff[len(vocab):] == eo[-1])                 # entries past the vocabulary hold its total length
    assert np.array_equal(vblob[:eo[-1]].astype(np.int64), eb.astype(np.int64))


def _edge_cases(seed):
    rng = random.Random(seed)
    ws = [chr(c) for c in SPACES]
    out = ["", " ", "\t\n", "".join(ws), "a", "ab", "aé", "a ab aé", " lead", "trail ", "  both  ", "dup dup dup x dup",
           "\U0001F600 smile \U0001F600", "\U00010000a \U0010FFFF", "a　b c d\x1ce", "\ud800 lone"]
    for c in ws:
        out += [c, f"x{c}y", f"{c}{c}z{c}"]
    alpha = ["a", "b", "ab", "ba", "é", "中", "\U0001F600", "z"] + ws
    for _ in range(200):
        out.append("".join(rng.choice(alpha) for _ in range(rng.randint(0, 20))))
    out.append(" ".join(f"t{rng.randint(0, 50)}" for _ in range(400)))               # hundreds of tokens
    return out


def test_edge_cases_two_lists_and_self_match():
    frm = _edge_cases(1)
    to = _edge_cases(2) + ["q" * 2500, "q" * 2500 + "r qq", "q" * 2499, "p" * 3000 + " " + "q" * 2500]   # tokens > 2 000 code points
    _check(frm, to)
    _check(to, frm)
    _check(frm)
    _check(to)
    _check(["", " "], ["a"])
    _check(["a"], ["", "　"])


def test_cjk_lists_with_many_code_points():
    rng = random.Random(3)
    cjk = [chr(0x4E00 + i) for i in range(600)]
    frm = [" ".join("".join(rng.choice(cjk) for _ in range(rng.randint(1, 4))) for _ in range(rng.randint(1, 5))) for _ in range(300)]
    to = [" ".join("".join(rng.choice(cjk) for _ in range(rng.randint(1, 4))) for _ in range(rng.randint(1, 5))) for _ in range(500)]
    _check(frm, to)


def test_movie_titles_and_company_names():
    from polyfuzz_b200 import datasets
    titles, _ = datasets.load_movie_titles()
    _check(titles["Netflix"], titles["IMDB"])
    names, _ = datasets.load_company_names()
    _check(names)
    _check(names[:5000], names[5000:])


# ---- the kept to-side -----------------------------------------------------------------------------------------------------
A = ["apple inc", "apples and pears", "the house", "similarity test", "new york jets", "Ålesund fc"]
T = ["apple", "apples inc", "mouse house", "the similar test", "new york giants", "jets of new york", "Ålesund", "zebra"]
B = ["pear apple", "unseen tokens here", "中文 apple", "ÿ house", "mouse", "jets jets new"]   # tokens / code points absent from A and T


def _matchers():
    from polyfuzz_b200 import EditDistance, RapidFuzz
    out = []
    for top_n in (1, 10):
        for scorer in ("WRatio", "token_set_ratio", "partial_ratio", "ratio"):
            out.append(lambda s=scorer, k=top_n: RapidFuzz(scorer=s, top_n=k))
        for scorer in ("ratio", "jaro_winkler", "dl"):
            for norm in (True, False):
                out.append(lambda s=scorer, k=top_n, nm=norm: EditDistance(scorer=s, normalize=nm, top_n=k))
    return out


@pytest.mark.parametrize("case", range(20))
def test_resident_equals_fresh(case):
    mk = _matchers()[case]
    m = mk()
    m.match(A, T)
    kept = m._kept().staged
    got = m.match(B, T, re_train=False)
    assert m._kept().staged is kept                            # scored against the kept to-side
    assert got.equals(mk().match(B, T))
    # an equal list that is another object is reused too
    assert m.match(B, list(T), re_train=False).equals(got) and m._kept().staged is kept
    # a self-match fit, then a transform of new strings against it
    m = mk()
    m.match(T)
    kept = m._kept().staged
    assert m.match(B, T, re_train=False).equals(got) and m._kept().staged is kept
    # a different or mutated to-list stages again
    T2 = T[:-1] + ["zebras"]
    assert m.match(B, T2, re_train=False).equals(mk().match(B, T2)) and m._kept().staged is not kept
    kept = m._kept().staged
    assert m.match(B, T[:-1], re_train=False).equals(mk().match(B, T[:-1])) and m._kept().staged is not kept
    T3 = list(T)
    m.match(B, T3)
    kept = m._kept().staged
    T3[1] = "apples inc."                                       # mutated in place after it was staged
    assert m.match(B, T3, re_train=False).equals(mk().match(B, T3)) and m._kept().staged is not kept
    # re_train=True always stages again
    kept = m._kept().staged
    m.match(B, T[:-1])
    assert m._kept().staged is not kept
    # pickling drops the device state; the first call after loading stages again
    m2 = pickle.loads(pickle.dumps(m))
    assert "_kept_targets" not in m2.__dict__
    assert m2.match(B, T[:-1], re_train=False).equals(mk().match(B, T[:-1]))


def test_resident_on_movie_titles():
    from polyfuzz_b200 import RapidFuzz, datasets
    titles, _ = datasets.load_movie_titles()
    to = titles["IMDB"][:20000]
    m = RapidFuzz(top_n=3)
    m.match(titles["Netflix"][:200], to)
    for lo in (200, 1200):
        new = titles["Netflix"][lo:lo + 300]
        pd.testing.assert_frame_equal(m.match(new, to, re_train=False), RapidFuzz(top_n=3).match(new, to))


def test_fit_transform_through_the_reference_orchestrator():
    if not os.path.isdir(os.path.join(REF, "polyfuzz")):
        pytest.skip("oracle/_ref (the byte-compiled reference orchestrator) was not built")
    os.environ["PFZ_REFERENCE_ROOT"] = REF
    from oracle import ref_shim
    ref_shim.REFERENCE_ROOT = REF
    ref_shim.install()
    from polyfuzz import PolyFuzz
    from polyfuzz_b200 import EditDistance, RapidFuzz
    for mk in (lambda: RapidFuzz(model_id="m"), lambda: EditDistance(model_id="m", normalize=False)):
        model = PolyFuzz(mk()).fit(A, T)
        kept = model.method._kept().staged
        out = model.transform(B)
        assert model.method._kept().staged is kept
        fresh = mk().match(B, T)
        assert out["EditDistance"].equals(fresh)
        model = PolyFuzz(mk()).fit(T)                           # self-match fit: its list is the to-list of transform
        kept = model.method._kept().staged
        assert model.transform(B)["EditDistance"].equals(fresh) and model.method._kept().staged is kept
