"""A numpy restatement of single linkage (polyfuzz/linkage.py:25-51) as parallel rounds: the rule K7 implements
(DESIGN.md 4.13), and the frames both the CPU and the GPU tests run it on.

The reference walks the kept rows with a dict m and a counter c = 0: if not m.get(F): (if not m.get(T): m[T] = m[F] = c;
c += 1 else: m[F] = m[T]).  Cluster id 0 is falsy and nonzero values never change, so with r0 the first kept row, key x is
nonzero before row p iff a kept row q in (r0, p) has F_q = x, or creates with T_q = x.  Row r0 creates; another row skips
when F is nonzero before it, else inherits when T is, else creates.  Here a round decides every row whose keys are known,
from the state at the start of the round, and the ids, the insertion order and the clusters follow from the outcomes."""
import numpy as np
import pandas as pd

INF = np.iinfo(np.int64).max
UNDEC, SKIP, INHERIT, CREATE = 1, 2, 3, 4


def outcomes(F, T, n_keys):
    """Row outcomes of kept rows F, T (key ids; r0 = row 0) by rounds.  Returns (status, firstF, createMin, rounds):
    firstF[x] = first row > 0 with F = x, createMin[x] = first create row > 0 with T = x (INF when none)."""
    n = len(F)
    status = np.full(n, UNDEC, dtype=np.int64)
    firstF = np.full(n_keys, INF, dtype=np.int64)
    createMin = np.full(n_keys, INF, dtype=np.int64)
    if n == 0:
        return status, firstF, createMin, 0
    status[0] = CREATE
    np.minimum.at(firstF, F[1:], np.arange(1, n))
    rounds = 0
    while True:
        p = np.flatnonzero(status == UNDEC)
        if p.size == 0:
            return status, firstF, createMin, rounds
        pend = np.full(n_keys, INF, dtype=np.int64)              # first undecided row per T key
        np.minimum.at(pend, T[p], p)
        f, t = F[p], T[p]
        f_set = (firstF[f] < p) | (createMin[f] < p)
        f_unset = ~f_set & (pend[f] >= p)
        t_set = (firstF[t] < p) | (createMin[t] < p)
        t_unset = ~t_set & (pend[t] >= p)
        new = np.select([f_set, f_unset & t_set, f_unset & t_unset], [SKIP, INHERIT, CREATE], UNDEC)
        assert new[0] != UNDEC                                  # the first undecided row always decides
        status[p] = new
        c = new == CREATE
        np.minimum.at(createMin, t[c], p[c])
        rounds += 1


def linkage_ids(F, T, n_keys):
    """(val, rank, rep, rounds) per key: final value, insertion rank and representative key (-1 when never written)."""
    n = len(F)
    status, firstF, createMin, rounds = outcomes(F, T, n_keys)
    val = np.full(n_keys, -1, dtype=np.int64)
    rank = np.full(n_keys, -1, dtype=np.int64)
    rep = np.full(n_keys, -1, dtype=np.int64)
    if n == 0:
        return val, rank, rep, rounds
    create = status == CREATE
    cid = np.cumsum(create) - 1                                 # create ids in row order
    set_at = np.minimum(firstF, createMin)                      # the row that first writes x nonzero
    ptr = np.arange(n)
    inh = status == INHERIT
    ptr[inh] = set_at[T[inh]]
    while True:                                                 # pointer jumping to the create row of each inherit chain
        nxt = ptr[ptr]
        if np.array_equal(nxt, ptr):
            break
        ptr = nxt
    keys = np.arange(n_keys)
    code = np.where(set_at < INF, 2 * np.minimum(set_at, n) + (createMin != set_at), -1)
    code[F[0]] = 1
    code[T[0]] = 0                                              # r0 writes T, then F
    written = code >= 0
    val[written] = np.where(set_at[written] < INF, cid[ptr[np.minimum(set_at[written], n - 1)]], 0)
    order = keys[written][np.argsort(code[written], kind="stable")]
    rank[order] = np.arange(order.size)
    first = {}
    for x in order:                                             # first key of each value, in insertion order
        first.setdefault(int(val[x]), int(x))
    rep[order] = [first[int(val[x])] for x in order]
    return val, rank, rep, rounds


def single_linkage(matches, min_similarity=0.8):
    """The three dicts of the reference's single_linkage, from linkage_ids."""
    kept = matches.loc[matches.Similarity > min_similarity, :]
    n = len(kept)
    codes, uniques = pd.factorize(pd.concat([kept["From"], kept["To"]], ignore_index=True))
    uniques = np.asarray(uniques, dtype=object)
    val, rank, rep, _ = linkage_ids(codes[:n].astype(np.int64), codes[n:].astype(np.int64), len(uniques))
    order = np.argsort(np.where(rank >= 0, rank, INF), kind="stable")[: int((rank >= 0).sum())]
    cluster_mapping = {uniques[x]: int(val[x]) for x in order}
    clusters = {}
    for x in order:
        clusters.setdefault(int(val[x]), []).append(uniques[x])
    cluster_name_map = {uniques[x]: uniques[rep[x]] for x in order}
    return clusters, cluster_mapping, cluster_name_map


def rounds_of(matches, min_similarity):
    kept = matches.loc[matches.Similarity > min_similarity, :]
    n = len(kept)
    codes, uniques = pd.factorize(pd.concat([kept["From"], kept["To"]], ignore_index=True))
    return outcomes(codes[:n].astype(np.int64), codes[n:].astype(np.int64), len(uniques))[3]


def as_lists(result):
    """The three dicts as lists of items: equal lists mean equal content and iteration order."""
    return [list(d.items()) for d in result]


# ---- frames -------------------------------------------------------------------------------------------------------------------
SCORES = np.array([0.5, 0.7, 0.75, 0.8, 0.9, 1.0])


def _frame(frm, to, sim):
    return pd.DataFrame({"From": list(frm), "To": list(to), "Similarity": np.asarray(sim, dtype=np.float64)})


def random_frame(rng, n, pool, unique_from=False, self_rate=0.0):
    """n rows over `pool` strings; Similarity from SCORES (0.75 among them, for thresholds equal to a score)."""
    names = np.array([f"s{i}" for i in range(max(pool, n if unique_from else 1))], dtype=object)
    frm = rng.permutation(names)[:n] if unique_from else names[rng.integers(0, pool, n)]
    to = names[rng.integers(0, pool, n)]
    same = rng.random(n) < self_rate
    to[same] = frm[same]
    return _frame(frm, to, SCORES[rng.integers(0, len(SCORES), n)])


def chain_frame(n, reverse=False):
    """s0 -> s1 -> s2 -> ... (each row waits for the one before it: one round per row), or its reverse."""
    a = [f"c{i}" for i in range(n + 1)]
    frm, to = (a[:-1], a[1:]) if not reverse else (a[1:], a[:-1])
    return _frame(frm, to, np.ones(n))


def hub_frame(rng, n, hubs=3):
    """n rows, almost all pointing at a few To strings."""
    frm = [f"h{i}" for i in range(n)]
    to = [f"hub{j}" for j in rng.integers(0, hubs, n)]
    return _frame(frm, to, np.ones(n))


def retarget_frame():
    """r0's keys written 0 and then re-targeted by later rows, as From and as To."""
    frm = ["a", "x", "b", "y", "z", "a", "w", "b"]
    to = ["b", "a", "y", "b", "a", "q", "x", "a"]
    return _frame(frm, to, np.ones(len(frm)))

