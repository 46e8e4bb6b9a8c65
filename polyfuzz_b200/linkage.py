"""K7 host driver: single linkage (polyfuzz/linkage.py:25-51) on the device, for PolyFuzz.group().

The kept rows' strings are mapped to key ids with one pd.factorize; the device decides every row's outcome, the cluster ids,
the insertion order of cluster_mapping and the grouping of `clusters` (include/pfz.h, pfz_linkage; DESIGN.md 4.13); the three
dicts are then built from four int32 arrays with vectorised gathers.  install_linkage() makes the unmodified PolyFuzz.group
use it."""
from typing import List, Mapping, Tuple

import numpy as np
import pandas as pd
import torch

from . import _lib
from .engine import _dev, _p, _stream, _to_dev, _ws


def linkage_arrays(F, T, n_keys, similarity=None, min_similarity=0.0):
    """Run K7 on int32 key ids F[n], T[n] in [0, n_keys).  With `similarity` (float64[n]) a row is kept when its score is
    > min_similarity (NaN is not kept); without it every row is kept.  Returns numpy (val, rank, rep, grouped, n_written):
    per key its final value, insertion rank and representative key (-1 when never written), and the written keys in the
    order of the reference's `clusters`."""
    F = np.ascontiguousarray(F, dtype=np.int32)
    T = np.ascontiguousarray(T, dtype=np.int32)
    n, n_keys = len(F), int(n_keys)
    if len(T) != n or (similarity is not None and len(similarity) != n):
        raise ValueError("F, T and similarity must have the same length")
    if n >= 1 << 30:
        raise ValueError("at most 2^30 - 1 rows")
    if n and (min(F.min(), T.min()) < 0 or max(F.max(), T.max()) >= n_keys):
        raise ValueError("key ids must lie in [0, n_keys)")
    dev = _dev()
    out = torch.full((4, max(n_keys, 1)), -1, dtype=torch.int32, device=dev)
    nw = torch.zeros(1, dtype=torch.int32, device=dev)
    if n:
        ws_bytes = int(_lib.load().pfz_linkage_ws_bytes(n, n_keys))
        # held until the launches are enqueued: a tensor freed earlier could hand its memory to the next allocation
        dF, dT, ws = _to_dev(F), _to_dev(T), _ws(ws_bytes)
        dS = None if similarity is None else _to_dev(np.asarray(similarity, dtype=np.float64))
        _lib.call("pfz_linkage", _p(dF), _p(dT), n, _p(dS), float(min_similarity), n_keys, _p(out[0]), _p(out[1]), _p(out[2]),
                  _p(out[3]), _p(nw), _p(ws), ws_bytes, _stream())
    host = out[:, :n_keys].cpu().numpy()
    return host[0], host[1], host[2], host[3], int(nw.item())


def _require_str(col, name):
    if len(col) and (col.isna().any() or pd.api.types.infer_dtype(col, skipna=False) != "string"):
        raise ValueError(f"single_linkage on the device needs str values in the kept rows' {name!r} column; "
                         "a kept row holds a null or a non-str value")


def single_linkage(matches: pd.DataFrame,
                   min_similarity: float = 0.8) -> Tuple[Mapping[int, List[str]], Mapping[str, int], Mapping[str, str]]:
    """Single linkage clustering from column 'From' to column 'To', on the device.

    The reference's `polyfuzz.linkage.single_linkage`, with its signature: the rows with Similarity > min_similarity are
    linked in frame order, and the three dicts it returns are equal to the reference's in content and iteration order.

    Arguments:
        matches: contains the columns *From*, *To*, and *Similarity* used for creating groups
        min_similarity: minimum similarity between strings before they can be merged into a group

    Returns:
        clusters: The populated clusters
        cluster_mapping: The mapping from a string to a cluster
        cluster_name_map: The mapping from a string to the representative string in its respective cluster

    Raises:
        ValueError: when a kept row's From or To is not a str.  That includes a null To, which only a negative
                    min_similarity keeps (the matchers give such rows a similarity of 0); the reference would use the
                    null itself as a key.
    """
    kept = matches.loc[matches.Similarity > min_similarity, :]
    frm, to = kept["From"], kept["To"]
    _require_str(frm, "From")
    _require_str(to, "To")
    n = len(kept)
    codes, uniques = pd.factorize(pd.concat([frm, to], ignore_index=True))
    uniques = np.asarray(uniques, dtype=object)
    val, rank, rep, grouped, nw = linkage_arrays(codes[:n], codes[n:], len(uniques))
    if nw == 0:
        return {}, {}, {}
    written = np.flatnonzero(rank >= 0)
    order = np.empty(nw, dtype=np.int64)
    order[rank[written]] = written                                   # keys in insertion order
    names = uniques[order].tolist()
    cluster_mapping = dict(zip(names, val[order].tolist()))
    cluster_name_map = dict(zip(names, uniques[rep[order]].tolist()))
    grouped = grouped[:nw]
    gval = val[grouped]
    starts = np.flatnonzero(np.r_[True, gval[1:] != gval[:-1]])       # each cluster is one run of `grouped`
    gnames = uniques[grouped].tolist()
    bounds = np.r_[starts, nw].tolist()
    clusters = {v: gnames[a:b] for v, a, b in zip(gval[starts].tolist(), bounds[:-1], bounds[1:])}
    return clusters, cluster_mapping, cluster_name_map


def install_linkage():
    """Make the unmodified PolyFuzz.group use this package's single_linkage: the name the orchestrator calls
    (polyfuzz/polyfuzz.py) and polyfuzz.linkage's own are rebound.  Kept apart from install(), which rebinds only the
    matcher classes."""
    import polyfuzz.linkage as pl
    import polyfuzz.polyfuzz as pp
    for mod in (pp, pl):
        mod.single_linkage = single_linkage
