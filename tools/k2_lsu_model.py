"""Developer tool: CPU model of the shared-memory traffic of the block kernel (spcos_blk3_kernel, 16-bit accumulators) on the
company-names self-match.  numpy + scipy + scikit-learn only; deterministic, no GPU.

    python tools/k2_lsu_model.py [--n 100000] [--tile 2048] [--rows 8] [--odd-tail] [--pair-loads] [--free-dump]

It rebuilds what the kernel walks: the TF-IDF matrix (sklearn vectoriser with the reference's analyzer), the to-index in
bank order (pfz_index_build with PFZ_INDEX_BANK_ORDER32: a segment of more than 32 postings is laid out in rounds that hold
every bank j mod 32 at most once, banks ascending), the from-row clustering key (ranks of the three heaviest terms), the
block tables (BF rows per block, split in two when the rows hold more than BF x 64 entries) and the work items (<= 32
postings of one term in one tile).  Then it counts per launch:

  * units (block, tile) and work items;
  * `red.shared.add` warp instructions, the ones that add 0 and their lane utilisation;
  * wavefronts per red: a red of a chunk costs the largest number of lanes that share a 4-byte bank -- the active lanes
    (bank = to-row mod 32; to-rows j and j + tile/2 share a word) plus the idle lanes, each in its dump word;
  * the scan (two 16-byte loads and two 16-byte stores per lane and warp step: 16 wavefronts) and the (row, weight)
    table loads (one wavefront each: every lane reads the same address).

Switches model the kernel changes one at a time:
  --odd-tail    an odd number of rows takes one red for the last entry (no red that adds 0);
  --pair-loads  the table is read with 16-byte loads, a list that starts on an odd entry (or ends on one) takes that entry
                with an 8-byte load (the start parity comes from the block table: terms ascending, rows ascending);
  --free-dump   idle lanes add into dump words in banks no active lane of the chunk uses.
"""
import argparse
import json
import os
import sys

import numpy as np
import scipy.sparse as sp

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

RANK_CAP = 16383
BANK_ORDER_MAX = 512


def tfidf_structure(n):
    from polyfuzz_b200 import datasets
    from oracle import tfidf
    names, kind = datasets.load_company_names(n)
    _, tf, _ = tfidf.fit_transform_sklearn(names)
    tf = sp.csr_matrix(tf)
    tf.sort_indices()
    return tf, kind


def cluster_order(tf, df):
    """blk_row_key_kernel + sort: rows by the ranks (df descending, term ascending) of their three heaviest terms, then row id."""
    n_vocab = tf.shape[1]
    order = np.lexsort((np.arange(n_vocab), -df))
    rank = np.empty(n_vocab, dtype=np.int64)
    rank[order] = np.minimum(np.arange(n_vocab), RANK_CAP)
    ip, ix = tf.indptr, tf.indices
    r3 = np.full((tf.shape[0], 3), RANK_CAP, dtype=np.int64)
    rr = rank[ix]
    for r in range(tf.shape[0]):
        x = np.sort(rr[ip[r]:ip[r + 1]])[:3]
        r3[r, :len(x)] = x
    return np.lexsort((np.arange(tf.shape[0]), r3[:, 2], r3[:, 1], r3[:, 0]))


def block_pairs(tf, perm, bf):
    """(block, term) pairs of the block tables: nf = rows of the block holding the term, start = the term's first entry in
    the block's (term, row) table.  A group of bf rows whose rows hold more than bf x 64 entries becomes two blocks."""
    nnz = np.diff(tf.indptr)[perm]
    n = len(perm)
    blk = np.empty(n, dtype=np.int64)
    nb = 0
    for p0 in range(0, n, bf):
        p1 = min(n, p0 + bf)
        if nnz[p0:p1].sum() <= bf * 64:
            blk[p0:p1] = nb; nb += 1
        else:
            h = min(p1, p0 + bf // 2)
            blk[p0:h] = nb; blk[h:p1] = nb + 1; nb += 2
    rows = np.repeat(np.arange(n), nnz)
    terms = tf[perm].indices.astype(np.int64)
    key = blk[rows] * tf.shape[1] + terms
    uk, nf = np.unique(key, return_counts=True)
    ublk = uk // tf.shape[1]
    first = np.r_[0, np.flatnonzero(np.diff(ublk)) + 1]
    cum = np.cumsum(nf) - nf
    start = cum - np.repeat(cum[first], np.diff(np.r_[first, len(uk)]))
    return nb, ublk, uk % tf.shape[1], nf, start


def chunk_stats(tf, tile):
    """Per term, summed over its (term, tile) segments: postings, work items, and the wavefronts of one red of each chunk,
    with idle lanes in their own dump word (bank = lane) and with idle lanes in free banks."""
    tc = tf.tocsc(); tc.sort_indices()
    n_vocab = tc.shape[1]
    term = np.repeat(np.arange(n_vocab), np.diff(tc.indptr))
    row = tc.indices.astype(np.int64)
    tl = row // tile
    j = row - tl * tile
    bank = j & 31
    seg = term * (tl.max() + 1) + tl                       # segments are contiguous, rows ascending (the fill order)
    segstart = np.r_[0, np.flatnonzero(np.diff(seg)) + 1]
    seglen = np.diff(np.r_[segstart, len(seg)])
    slen = np.repeat(seglen, seglen)
    pos_in = np.arange(len(seg)) - np.repeat(segstart, seglen)
    # bank order: rank within (segment, bank) in fill order, then banks ascending inside a round
    sb = seg * 32 + bank
    o = np.lexsort((pos_in, sb))
    sbo = sb[o]
    gst = np.r_[0, np.flatnonzero(np.diff(sbo)) + 1]
    rk = np.empty(len(seg), dtype=np.int64)
    rk[o] = np.arange(len(seg)) - np.repeat(gst, np.diff(np.r_[gst, len(seg)]))
    reorder = (slen > 32) & (slen <= BANK_ORDER_MAX)
    k2 = np.where(reorder, rk * 32 + bank, pos_in)
    o2 = np.lexsort((k2, seg))
    pos = np.empty(len(seg), dtype=np.int64)
    pos[o2] = np.arange(len(seg)) - np.repeat(segstart, seglen)  # position in the segment after the arrangement
    chunk_of = np.repeat(segstart, seglen) + (pos // 32) * 32   # global id of the posting's chunk (its first slot)
    cid, inv = np.unique(chunk_of, return_inverse=True)
    counts = np.zeros((len(cid), 32), dtype=np.int32)
    np.add.at(counts, (inv, bank), 1)
    cnt = counts.sum(1)
    w_act = counts.max(1)
    idle = (np.arange(32)[None, :] >= cnt[:, None]).astype(np.int32)
    w_dump = (counts + idle).max(1)
    cterm = term[cid]
    out = {
        "postings": np.bincount(term, minlength=n_vocab).astype(np.float64),
        "chunks": np.bincount(cterm, minlength=n_vocab).astype(np.float64),
        "w_dump": np.bincount(cterm, weights=w_dump, minlength=n_vocab),
        "w_act": np.bincount(cterm, weights=w_act, minlength=n_vocab),
    }
    return out, int(tl.max() + 1)


def model(n=100_000, tile=2048, bf=8, odd_tail=False, pair_loads=False, free_dump=False, _cache={}):
    key = (n, tile, bf)
    if key not in _cache:
        tf, kind = tfidf_structure(n)
        df = np.bincount(tf.indices, minlength=tf.shape[1]).astype(np.float64)
        perm = cluster_order(tf, df)
        nb, _ublk, uterm, nf, start = block_pairs(tf, perm, bf)
        cs, n_tiles = chunk_stats(tf, tile)
        _cache[key] = (kind, n_tiles, nb, uterm, nf, start, cs, tf.shape[0])
    kind, n_tiles, nb, uterm, nf, start, cs, n_rows = _cache[key]
    C = cs["chunks"][uterm]                                  # items of the (block, term) pair over all tiles
    Pp = cs["postings"][uterm]
    W = (cs["w_act"] if free_dump else cs["w_dump"])[uterm]  # wavefronts of one red, summed over the pair's chunks
    nf = nf.astype(np.float64)
    reds_per_item = nf if odd_tail else 2 * np.ceil(nf / 2)
    dead_per_item = np.zeros_like(nf) if odd_tail else (nf % 2)
    if pair_loads:
        peel = (start % 2 == 1).astype(np.float64)
        rest = nf - peel
        loads_per_item = peel + np.floor(rest / 2) + (rest % 2)
    else:
        loads_per_item = 2 * np.ceil(nf / 2)
    reds = float((reds_per_item * C).sum())
    useful = float((nf * Pp).sum())
    red_wf = float((reds_per_item * W).sum())
    scan_steps = float(n_rows) * n_tiles * (tile // 2 * 4 // 1024)
    res = {
        "data": kind, "n": n_rows, "tile": tile, "rows_per_block": bf, "n_tiles": n_tiles, "blocks": nb,
        "switches": {"odd_tail": odd_tail, "pair_loads": pair_loads, "free_dump": free_dump},
        "units": nb * n_tiles,
        "items": float(C.sum()),
        "block_term_pairs": int(len(nf)), "frac_pairs_nf1": float((nf == 1).mean()),
        "red_instr": reds, "red_add_zero": float((dead_per_item * C).sum()),
        "red_lane_util": useful / (32.0 * reds),
        "red_wavefronts": red_wf, "wavefronts_per_red": red_wf / reds,
        "table_loads": float((loads_per_item * C).sum()),
        "scan_steps": scan_steps, "scan_wavefronts": 16.0 * scan_steps,
    }
    res["lsu_wavefronts"] = res["red_wavefronts"] + res["table_loads"] + res["scan_wavefronts"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--tile", type=int, default=2048)
    ap.add_argument("--rows", type=int, default=8)
    ap.add_argument("--odd-tail", action="store_true")
    ap.add_argument("--pair-loads", action="store_true")
    ap.add_argument("--free-dump", action="store_true")
    ap.add_argument("--all", action="store_true", help="the old layout and each change added in turn")
    a = ap.parse_args()
    if a.all:
        steps = [("old layout", {}), ("+ odd tail", {"odd_tail": True}), ("+ paired loads", {"odd_tail": True, "pair_loads": True}),
                 ("+ free dump banks", {"odd_tail": True, "pair_loads": True, "free_dump": True})]
        base = None
        for name, kw in steps:
            r = model(a.n, a.tile, a.rows, **kw)
            base = base or r["lsu_wavefronts"]
            print(f"{name:20s} reds {r['red_instr']:.3e} (add 0: {r['red_add_zero']:.2e}, lanes {r['red_lane_util']:.2f})  "
                  f"wf/red {r['wavefronts_per_red']:.2f}  red wf {r['red_wavefronts']:.3e}  table loads {r['table_loads']:.3e}  "
                  f"scan wf {r['scan_wavefronts']:.3e}  total wf {r['lsu_wavefronts']:.3e} ({r['lsu_wavefronts'] / base:.3f})")
        print(json.dumps(r))
    else:
        print(json.dumps(model(a.n, a.tile, a.rows, a.odd_tail, a.pair_loads, a.free_dump)))


if __name__ == "__main__":
    main()
