"""Host logic of the kept to-side of RapidFuzz / EditDistance (CPU only, the kernels stubbed): a re_train=False call whose
to-list equals the kept one stages only the from-list; a different, mutated or re-trained to-list stages again; pickling
drops the kept state; and at world size 2 over gloo each rank keeps its own shard."""
import os
import pickle
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
FROM = ["apple pie", "apples", "house of cards", "recal", "similarity"]
TO = ["apple", "apples inc", "mouse house", "cards house", "similar"]


class _Lib:
    def __init__(self):
        self.names = []

    def call(self, name, *args):
        self.names.append(name)


def _cpu_stubs(monkeypatch, mod):
    lib = _Lib()
    monkeypatch.setattr(mod, "_lib", lib)
    monkeypatch.setattr(mod, "_dev", lambda: torch.device("cpu"))
    monkeypatch.setattr(mod, "_to_dev", lambda arr, dtype=None: (torch.from_numpy(np.ascontiguousarray(arr)) if dtype is None
                                                                else torch.from_numpy(np.ascontiguousarray(arr)).view(dtype)))
    monkeypatch.setattr(mod, "_blob_to_dev", lambda b: torch.from_numpy(np.ascontiguousarray(b).astype(np.int64)))
    monkeypatch.setattr(mod, "_stream", lambda: None)
    monkeypatch.setattr(mod, "_p", lambda t: None)
    return lib


def test_token_tables_of_an_equal_to_list_are_not_rebuilt(monkeypatch):
    from polyfuzz_b200 import editdist, fuzzy
    lib = _cpu_stubs(monkeypatch, fuzzy)
    kept = editdist.KeptTargets()

    def sides(frm, to, reuse):
        lib.names.clear()
        fuzzy._enqueue(frm, to, "WRatio", 0.0, to is frm, None, 0, 0, None, kept, reuse)
        return lib.names.count("pfz_tok_side")

    assert sides(FROM, TO, False) == 2                         # both lists
    staged = kept.staged
    assert sides(["new strings"], list(TO), True) == 1         # only the from-list; the kept to-side serves
    assert kept.staged is staged
    assert sides(["new strings"], TO, False) == 2 and kept.staged is not staged     # re_train=True stages again
    staged = kept.staged
    assert sides(["new strings"], TO[:-1] + ["other"], True) == 2 and kept.staged is not staged
    lst = list(TO)
    assert sides(FROM, lst, False) == 2
    lst[0] = "changed"                                          # mutated after it was staged
    assert sides(FROM, lst, True) == 2
    assert sides(TO, TO, False) == 1                            # self-match: one shared side ...
    assert sides(FROM, list(TO), True) == 1                     # ... which a transform against the same list reuses
    assert kept.key[0] == ("k3b", 0)


def test_edit_targets_of_an_equal_to_list_are_not_rebuilt(monkeypatch):
    from polyfuzz_b200 import EditDistance, RapidFuzz, editdist
    _cpu_stubs(monkeypatch, editdist)
    made = []
    real = editdist.EditTargets
    monkeypatch.setattr(editdist, "EditTargets", lambda lst: made.append(len(lst)) or real(lst))
    for m in (RapidFuzz(scorer="ratio"), EditDistance(normalize=False), RapidFuzz(scorer="levenshtein", top_n=3)):
        made.clear()
        m.match(FROM, TO)
        m.match(["x"], list(TO), re_train=False)
        m.match(["y"], TO, re_train=False)
        assert made == [len(TO)]
        m.match(["y"], TO)                                      # re_train=True (the default) stages again
        m.match(["y"], TO[:3], re_train=False)                  # so does another list
        assert made == [len(TO)] * 2 + [3]
        made.clear()
        m.match(TO)                                             # PolyFuzz.fit(to) then transform(new)
        m.match(["z"], TO, re_train=False)
        assert made == [len(TO)]
        m2 = pickle.loads(pickle.dumps(m))                      # the device state is not pickled
        assert "_kept_targets" not in m2.__dict__
        m2.match(["z"], TO, re_train=False)
        assert made == [len(TO)] * 2


def test_token_scorers_pass_the_kept_state(monkeypatch):
    from polyfuzz_b200 import RapidFuzz, fuzzy
    seen = []

    def fake(frm, to, *a, kept=None, reuse=False, **kw):
        seen.append(kept.stage(("k3b", 0), to, lambda lst: object(), reuse))
        n = len(frm)
        shape = (n,) if len(a) < 1 or not isinstance(a[0], int) else (n, a[0])
        return torch.full(shape, -1, dtype=torch.int32), torch.zeros(shape, dtype=torch.float64)

    monkeypatch.setattr(fuzzy, "fuzz_argbest", fake)
    m = RapidFuzz()
    m.match(FROM, TO)
    m.match(["x"], TO, re_train=False)
    m.match(["x"], TO)
    assert seen[0] is seen[1] and seen[2] is not seen[1]


# ---- distributed=True at world size 2 over gloo: each rank keeps its own shard ---------------------------------------------
def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from polyfuzz_b200 import RapidFuzz, editdist
        from polyfuzz_b200.distributed import shard_bounds
        from polyfuzz_b200.matchers import _rapidfuzz
        made = []
        editdist.EditQueries = lambda lst: lst
        editdist.EditTargets = lambda lst: made.append(list(lst)) or list(lst)

        def staged(Q, T, metric, cutoff, self_shift=0, to_index_base=0, **kw):
            n = len(Q)
            return (torch.full((n,), -1, dtype=torch.int32), torch.zeros(n, dtype=torch.float64), torch.full((n,), -1, dtype=torch.int32))
        editdist.edit_argbest_staged = staged
        _rapidfuzz.editdist.lev_merge = lambda gi, gs, gd: (gi[0], gs[0], gd[0])
        to = TO + ["house", "apple pies"]
        lo, hi = shard_bounds(len(to), world, rank)
        m = RapidFuzz(scorer="ratio", distributed=True)
        m.match(FROM, to)
        m.match(["new"], list(to), re_train=False)
        assert made == [to[lo:hi]], made
        m.match(["new"], to)
        assert made == [to[lo:hi]] * 2 and m._kept().key[0] == ("k3", lo)
        out.put((rank, "ok"))
    except Exception:  # pragma: no cover
        import traceback
        out.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo_each_rank_keeps_its_shard():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res
