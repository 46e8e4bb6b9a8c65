"""CPU tests of the host logic of RapidFuzz / EditDistance with top_n (frame layout, clipping, empty slots, score scaling,
EditDistance's joint normalisation, which entry point runs, argument checks), with the device entry points replaced by numpy
stand-ins -- the kernels themselves are covered by tests/test_gpu_editdist_topn.py -- and the distributed path at world size 2
over gloo."""
import os
import sys

import numpy as np
import pandas as pd
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
FROM = ["apple", "apples", "appl", "recal", "house", "similarity"]
TO = ["apple", "apples", "mouse"]


def fake_scores(frm, to):
    """A stand-in scorer in [0, 100] with ties: 100 - 10 * |len(a) - len(b)| - 5 * (first letters differ), floored at 0."""
    return np.array([[max(0.0, 100.0 - 10 * abs(len(a) - len(b)) - 5 * (a[:1] != b[:1])) for b in to] for a in frm])


def fake_rank(frm, to, k, cutoff, exclude_self, self_shift=0, to_index_base=0):
    S = fake_scores(frm, to)
    oi = np.full((len(frm), k), -1, np.int32); ov = np.zeros((len(frm), k))
    for i in range(len(frm)):
        c = np.array([j for j in range(len(to)) if S[i, j] >= cutoff and not (exclude_self and j == i + self_shift)], dtype=np.int64)
        if len(c):
            c = c[np.lexsort((c, -S[i, c]))][:k]
            oi[i, :len(c)] = c + to_index_base; ov[i, :len(c)] = S[i, c]
    return oi, ov


class Stubs:
    """Numpy stand-ins for editdist.edit_argbest / edit_topk and fuzzy.fuzz_argbest / fuzz_topk that record their calls."""

    def __init__(self):
        self.calls = []

    def edit_argbest(self, frm, to, metric="ratio", score_cutoff=0.0, exclude_self=False, **kw):
        self.calls.append(("edit_argbest", metric, 1))
        i, v = fake_rank(frm, to, 1, score_cutoff, exclude_self)
        return torch.from_numpy(i[:, 0].copy()), torch.from_numpy(v[:, 0].copy()), torch.zeros(len(frm), dtype=torch.int32)

    def edit_topk(self, frm, to, k, metric="ratio", score_cutoff=0.0, exclude_self=False, **kw):
        self.calls.append(("edit_topk", metric, k))
        i, v = fake_rank(frm, to, k, score_cutoff, exclude_self)
        return torch.from_numpy(i), torch.from_numpy(v)

    def fuzz_argbest(self, frm, to, scorer="WRatio", score_cutoff=0.0, exclude_self=False, **kw):
        self.calls.append(("fuzz_argbest", scorer, 1))
        i, v = fake_rank(frm, to, 1, score_cutoff, exclude_self)
        return torch.from_numpy(i[:, 0].copy()), torch.from_numpy(v[:, 0].copy())

    def fuzz_topk(self, frm, to, k, scorer="WRatio", score_cutoff=0.0, exclude_self=False, **kw):
        self.calls.append(("fuzz_topk", scorer, k))
        i, v = fake_rank(frm, to, k, score_cutoff, exclude_self)
        return torch.from_numpy(i), torch.from_numpy(v)


@pytest.fixture
def stubs(monkeypatch):
    from polyfuzz_b200 import editdist, fuzzy
    s = Stubs()
    for mod, name in ((editdist, "edit_argbest"), (editdist, "edit_topk"), (fuzzy, "fuzz_argbest"), (fuzzy, "fuzz_topk")):
        monkeypatch.setattr(mod, name, getattr(s, name))
    return s


def _names(k):
    out = ["From"]
    for r in range(k):
        out += ["To", "Similarity"] if r == 0 else [f"To_{r + 1}", f"Similarity_{r + 1}"]
    return out


@pytest.mark.parametrize("k", [1, 2, 5])
def test_columns_clipping_and_entry_points(stubs, k):
    from polyfuzz_b200 import EditDistance, RapidFuzz
    to = TO + ["mouse", "houses", "apply"]                            # 5 distinct to-strings
    for scorer, entry in (("WRatio", "fuzz"), ("ratio", "edit"), ("levenshtein", "edit")):
        stubs.calls.clear()
        df = RapidFuzz(scorer=scorer, top_n=k).match(FROM, to)
        assert list(df.columns) == _names(k)
        assert stubs.calls == [(f"{entry}_argbest" if k == 1 else f"{entry}_topk", {"levenshtein": "norm_lev"}.get(scorer, scorer), k)]
    stubs.calls.clear()
    df = EditDistance(scorer="jaro_winkler", top_n=k).match(FROM, to)
    assert list(df.columns) == _names(k) and stubs.calls == [("edit_argbest" if k == 1 else "edit_topk", "jaro_winkler", k)]
    # clipped to len(set(to_list)) = 2 when a to_list is given
    stubs.calls.clear()
    df = RapidFuzz(scorer="ratio", top_n=k).match(FROM, ["apple", "mouse", "apple"])
    assert list(df.columns) == _names(min(k, 2)) and stubs.calls[0][2] == min(k, 2)
    # top_n clipped to 1 runs the arg-best path and gives the top-1 frame
    stubs.calls.clear()
    df = RapidFuzz(scorer="ratio", top_n=k).match(FROM, ["apple", "apple"])
    assert stubs.calls == [("edit_argbest", "ratio", 1)] and list(df.columns) == _names(1)
    # a self-match is not clipped
    stubs.calls.clear()
    df = EditDistance(normalize=False, top_n=k).match(["a", "b"])
    assert list(df.columns) == _names(k) and stubs.calls[0][2] == k


def test_empty_slots_scaling_and_first_columns(stubs):
    from polyfuzz_b200 import EditDistance, RapidFuzz
    frm = ["abc", "abcd", "zz"]
    to = ["abd", "xbcd", "abcde", "q"]
    df = RapidFuzz(scorer="ratio", score_cutoff=0.9, top_n=3).match(frm, to)
    i, v = fake_rank(frm, to, 3, 90.0, False)
    for r, (tc, sc) in enumerate((("To", "Similarity"), ("To_2", "Similarity_2"), ("To_3", "Similarity_3"))):
        assert df[tc].tolist() == [to[j] if j >= 0 else None for j in i[:, r]]
        assert df[sc].tolist() == [x / 100 if j >= 0 else 0.0 for x, j in zip(v[:, r], i[:, r])]
    assert df["To_3"].isna().any() and df["Similarity"].dtype == np.float64
    # levenshtein is 0..1 already: not divided by 100
    df = RapidFuzz(scorer="levenshtein", top_n=2).match(frm, to)
    assert df["Similarity"].tolist() == fake_rank(frm, to, 2, 0.0, False)[1][:, 0].tolist()
    # the first three columns of a top_n = k frame are the top_n = 1 frame
    pd.testing.assert_frame_equal(RapidFuzz(scorer="ratio", score_cutoff=0.9, top_n=3).match(frm, to)[["From", "To", "Similarity"]],
                                  RapidFuzz(scorer="ratio", score_cutoff=0.9).match(frm, to))
    pd.testing.assert_frame_equal(EditDistance(normalize=False, top_n=3).match(frm, to)[["From", "To", "Similarity"]],
                                  EditDistance(normalize=False).match(frm, to))


def test_editdistance_joint_normalisation_skips_empty_slots(stubs):
    from polyfuzz_b200 import EditDistance
    frm = ["a", "bb", "ccc"]                                          # self-match, top_n = 3: each row has 2 candidates
    raw = EditDistance(normalize=False, top_n=3).match(frm)
    df = EditDistance(top_n=3).match(frm)
    cols = ["Similarity", "Similarity_2", "Similarity_3"]
    r = raw[cols].to_numpy(); filled = raw[["To", "To_2", "To_3"]].notna().to_numpy()
    assert not filled[:, 2].any() and filled[:, :2].all()
    lo, hi = r[filled].min(), r[filled].max()
    exp = np.where(filled, (r - lo) / (hi - lo), 0.0)
    np.testing.assert_array_equal(df[cols].to_numpy(), exp)
    assert df["Similarity"].max() == 1.0 and df[cols].to_numpy()[filled].min() == 0.0 and (df["Similarity_3"] == 0.0).all()


@pytest.mark.parametrize("bad", [0, 33, 2.5, "3", -1, True, None])
def test_top_n_is_checked_before_any_work(stubs, bad):
    from polyfuzz_b200 import EditDistance, RapidFuzz
    for cls in (RapidFuzz, EditDistance):
        with pytest.raises(ValueError, match="1 to 32"):
            cls(top_n=bad)
    assert stubs.calls == []
    from polyfuzz_b200 import editdist, fuzzy
    assert editdist.check_top_n(32) == 32 and editdist.check_top_n(np.int64(3)) == 3
    with pytest.raises(ValueError, match="1 to 32"):
        fuzzy.check_top_n(bad)


# ---- distributed=True at world size 2 over gloo ----------------------------------------------------------------------------
def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle import native
        from polyfuzz_b200 import EditDistance, RapidFuzz, editdist, fuzzy
        from polyfuzz_b200.matchers import _rapidfuzz
        seen = []

        def shard_topk(frm, to, k, metric="ratio", score_cutoff=0.0, exclude_self=False, self_shift=0, to_index_base=0, **kw):
            seen.append((len(to), self_shift, to_index_base))
            i, v = fake_rank(frm, to, k, score_cutoff, exclude_self, self_shift, to_index_base)
            return torch.from_numpy(i), torch.from_numpy(v)

        def merge(gi, gv, k):                                          # the CPU oracle of pfz_topk_merge (same key)
            mi, mv = native.topk_merge(gi.numpy(), gv.numpy(), k)
            return torch.from_numpy(mi), torch.from_numpy(mv)
        fuzzy.fuzz_topk = shard_topk
        editdist.EditQueries = lambda lst: lst
        editdist.EditTargets = lambda lst: lst
        editdist.edit_topk_staged = lambda Q, T, k, metric, cutoff, **kw: shard_topk(Q, T, k, metric, cutoff, **kw)
        _rapidfuzz.merge_topk_any = merge
        frm = FROM + ["apple", "mouses", "hose"]
        to = TO + ["house", "apple", "similar", "app"]
        for matcher, single in ((RapidFuzz(top_n=4, distributed=True), fake_rank(frm, to, 4, 0.0, False)),
                                (EditDistance(scorer="ratio", normalize=False, top_n=4, distributed=True), fake_rank(frm, to, 4, float("-inf"), False)),
                                (RapidFuzz(scorer="ratio", top_n=5, distributed=True), None)):
            if single is None:                                          # self-match: to-row i + self_shift excluded on its shard
                df = matcher.match(frm)
                single = fake_rank(frm, frm, 5, 0.0, True)
                targets = frm
            else:
                df = matcher.match(frm, to)
                targets = to
            k = single[0].shape[1]
            to_cols = ["To"] + [f"To_{r + 1}" for r in range(1, k)]
            assert [df[c].tolist() for c in to_cols] == [[targets[j] if j >= 0 else None for j in single[0][:, r]] for r in range(k)]
        lo = 0 if rank == 0 else 4                                     # shard_bounds(7, 2, rank) of the two-list calls
        assert seen[0] == (len(to[lo:lo + 4]), -lo, lo) and seen[2][1:] == (-(0 if rank == 0 else 5), 0 if rank == 0 else 5)
        out.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        import traceback
        out.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo_distributed_top_n():
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = 31500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    res = [out.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res
