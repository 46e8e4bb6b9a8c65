"""Host oracle of K3b's token tables (include/pfz.h, pfz_tok_*): the Python derivation fuzzy.py ran before the tables were
built on the device, kept as the reference the device buffers are compared against.

Tokens are str.split()'s; one dictionary numbers the distinct tokens of both lists in sorted (Python string) order; per string
S(s) joins all its tokens in that order, U(s) the distinct ones, and the signature ORs one bit per distinct id."""
import numpy as np


def derive(strings):
    toks = [s.split() for s in strings]
    return toks, [" ".join(sorted(t)) for t in toks], [" ".join(sorted(set(t))) for t in toks]


def _cps(strings):
    """UTF-32 blob (int32) + int64 offsets of a list, the device layout."""
    off = np.zeros(len(strings) + 1, dtype=np.int64)
    np.cumsum([len(s) for s in strings], out=off[1:])
    blob = np.frombuffer("".join(strings).encode("utf-32-le", "surrogatepass"), dtype=np.uint32).astype(np.int32)
    return blob, off


def side_tables(strings, toks, sorted_joined, uniq_joined, tok_id):
    """One list's tables: s / S / U as (blob, offsets), tok_ptr, tok_ids, sig (uint64), n_all."""
    n = len(strings)
    ptr = np.zeros(n + 1, dtype=np.int32)
    ids, sig = [], np.zeros(n, dtype=np.uint64)
    n_all = np.zeros(n, dtype=np.int32)
    for i, t in enumerate(toks):
        u = sorted({tok_id[x] for x in t})
        ids.extend(u)
        ptr[i + 1] = ptr[i] + len(u)
        n_all[i] = len(t)
        b = 0
        for x in u:
            b |= 1 << (((x * 0x9E3779B1) >> 13) & 63)
        sig[i] = b
    return {"s": _cps(strings), "S": _cps(sorted_joined), "U": _cps(uniq_joined), "tok_ptr": ptr,
            "tok_ids": np.asarray(ids, dtype=np.int32), "sig": sig, "n_all": n_all}


def tables(from_list, to_list=None):
    """(from tables, to tables, vocabulary) for a two-list call, or a self-match when to_list is None (one shared side)."""
    ftoks, fS, fU = derive(from_list)
    if to_list is None:
        ttoks = []
    else:
        ttoks, tS, tU = derive(to_list)
    vocab = sorted({x for t in ftoks for x in t} | {x for t in ttoks for x in t})
    tok_id = {x: i for i, x in enumerate(vocab)}
    F = side_tables(from_list, ftoks, fS, fU, tok_id)
    T = F if to_list is None else side_tables(to_list, ttoks, tS, tU, tok_id)
    return F, T, vocab
