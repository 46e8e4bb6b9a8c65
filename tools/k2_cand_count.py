"""Developer tool (CPU only): how many candidates the block kernel's filter queues per from-row, under three rules for
the gate a row starts from, on the headline data (100k company names, TF-IDF trigrams, self-match, top-10).

    python tools/k2_cand_count.py [--rows 1500] [--tile 4096] [--k 10] [--budget 128,256] [--seeds 32]

The model follows spcos_blk3_kernel in 16-bit mode (DESIGN §4.1) with exact scores in place of the fixed-point sums:
unit 2^-15, margin MQ = 4 m + 2 for a row of m terms, tiles of --tile to-rows visited in order, and in each tile the cells
scanned 16-byte group by group (to-rows j and j + tile/2 share word j; a group holds four words).  A cell is queued when its
sum is above the gate; after each group with a queued cell the gate rises to (K-th largest queued sum - MQ); while fewer
than K sums have been queued and the row is not seeded, each tile first raises the gate to (K-th of the 32 lane maxima - MQ).
The diagonal never competes.  Gate at the start of the row:
  * today:   the min_similarity threshold (0 here);
  * seeded:  a seed pass run before the main kernel (DESIGN §4.1 reports one that was built and timed) -- partial dot
             products over the row's rarest terms (ascending document frequency, while their postings fit in --budget), the
             --seeds to-rows with the largest partial sums scored exactly, and floor(kv * 2^15 - MQ) from the K-th eligible
             exact score kv (0 with fewer than K eligible).  kv is a lower bound of the row's final K-th score, so the
             results do not change;
  * perfect: the same expression from the row's true K-th score (only the margin band is left).
Also reported: the postings the seed pass reads, against P (every posting every from-row visits).
The GPU's own count is the block kernel's gcnt array, which tools/k2_breakdown.py reports.
"""
import argparse
import json
import os
import sys

import numpy as np
import scipy.sparse as sp

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000, help="company names (the headline size)")
    ap.add_argument("--names", default=None, help="JSON file of names (a list, or {'names': [...]}) instead of the company names")
    ap.add_argument("--rows", type=int, default=1500, help="random from-rows simulated")
    ap.add_argument("--tile", type=int, default=4096)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--budget", default="64,128,256,512", help="seed pass posting budgets per row (comma-separated)")
    ap.add_argument("--seeds", default="32", help="to-rows scored exactly per row (comma-separated, <= 32)")
    ap.add_argument("--seed", type=int, default=0, help="random seed of the row sample")
    return ap.parse_args()


def scan_row(cells, scores, m, T, K, gate0, seeded):
    """Candidates queued by one row.  cells: to-rows with a non-zero score (diagonal removed), scores: exact scores."""
    MQ = 4 * m + 2
    sums = scores * 32768.0
    half = T // 2
    gate, top = float(gate0), []                       # top: the K largest queued sums, descending
    n_q = 0
    tiles = cells // T
    for tau in np.unique(tiles):
        sel = tiles == tau
        jl = cells[sel] - tau * T
        s = sums[sel]
        word = jl % half
        grp = word // 4
        if len(top) < K and not seeded:                # lane maxima: lane l holds the groups c = l (mod 32)
            lm = np.zeros(32)
            np.maximum.at(lm, grp % 32, s)
            kth = np.sort(lm)[::-1][K - 1]
            if kth > MQ:
                gate = max(gate, kth - MQ)
        keep = s > gate
        if not keep.any():
            continue
        order = np.lexsort(((word % 4) * 2 + (jl >= half), grp))
        order = order[keep[order]]
        g_prev, hit = None, False
        for i in order:
            g = grp[i]
            if g != g_prev and hit and len(top) >= K:
                gate = max(gate, top[K - 1] - MQ)      # the gate rises after each group with a queued cell
            if g != g_prev:
                hit = False
            g_prev = g
            if s[i] > gate:
                n_q += 1
                hit = True
                top.append(s[i]); top.sort(reverse=True); del top[K:]
    return n_q


def kth_gate(kv, m):
    y = kv * 32768.0 - (4 * m + 2)
    return 0.0 if y <= 0.0 else float(np.floor(y))


def main():
    args = parse()
    from polyfuzz_b200 import datasets
    from oracle import tfidf as otfidf
    if args.names:
        names = json.load(open(args.names))
        names, kind = (names["names"] if isinstance(names, dict) else names), os.path.basename(args.names)
    else:
        names, kind = datasets.load_company_names(args.n, seed=0)
    X, _, _ = otfidf.fit_transform_sklearn(names)
    X = sp.csr_matrix(X, dtype=np.float64); X.sort_indices()
    n, K, T = X.shape[0], args.k, args.tile
    df = np.diff(X.tocsc().indptr)                     # document frequency of every term in the to-side (= from-side)
    XT = X.T.tocsr()
    P = float(np.sum(df[X.indices]))
    rng = np.random.default_rng(args.seed)
    rows = np.sort(rng.choice(n, size=min(args.rows, n), replace=False))
    budgets = [int(b) for b in args.budget.split(",")]
    dseeds = [int(d) for d in args.seeds.split(",")]
    res = {"data": kind, "n": n, "rows": len(rows), "tile": T, "k": K, "P_postings": P,
           "today": [], "perfect": [], "seeded": {f"B{b}_D{d}": [] for b in budgets for d in dseeds},
           "seed_postings": {f"B{b}": [] for b in budgets}}
    for c0 in range(0, len(rows), 100):
        blk = rows[c0:c0 + 100]
        S = (X[blk] @ X.T).tocsr()
        for q, r in enumerate(blk):
            a0, a1 = X.indptr[r], X.indptr[r + 1]
            m = a1 - a0
            cols, vals = S.indices[S.indptr[q]:S.indptr[q + 1]], S.data[S.indptr[q]:S.indptr[q + 1]]
            nd = cols != r
            cols, vals = cols[nd], vals[nd]
            o = np.argsort(cols); cols, vals = cols[o], vals[o]
            res["today"].append(scan_row(cols, vals, m, T, K, 0.0, False))
            top = np.sort(vals)[::-1]
            kv_true = top[K - 1] if len(top) >= K else 0.0
            g = kth_gate(kv_true, m) if len(top) >= K else 0.0
            res["perfect"].append(scan_row(cols, vals, m, T, K, g, g > 0))
            terms, w = X.indices[a0:a1], X.data[a0:a1]
            by_df = np.argsort(df[terms], kind="stable")
            cum = np.cumsum(df[terms][by_df])
            for b in budgets:
                light = by_df[cum <= b]
                res["seed_postings"][f"B{b}"].append(int(cum[len(light) - 1]) if len(light) else 0)
                part = {}
                for e in light:                        # partial dot products over the light terms
                    t = terms[e]
                    for p in range(XT.indptr[t], XT.indptr[t + 1]):
                        j = XT.indices[p]
                        part[j] = part.get(j, 0.0) + w[e] * XT.data[p]
                for d in dseeds:
                    best = sorted(part.items(), key=lambda x: (-x[1], x[0]))[:d]
                    sc = sorted([S[q, j] for j, _ in best if j != r and S[q, j] > 0.0], reverse=True)
                    gs = kth_gate(sc[K - 1], m) if len(sc) >= K else 0.0
                    res["seeded"][f"B{b}_D{d}"].append(scan_row(cols, vals, m, T, K, gs, gs > 0))
    out = {"data": kind, "n": n, "rows": len(rows), "tile": T, "k": K, "P_postings": P,
           "today_mean": float(np.mean(res["today"])), "today_max": int(np.max(res["today"])),
           "perfect_mean": float(np.mean(res["perfect"])), "seeded": {}}
    for b in budgets:
        sp_mean = float(np.mean(res["seed_postings"][f"B{b}"]))
        for d in dseeds:
            c = res["seeded"][f"B{b}_D{d}"]
            out["seeded"][f"B{b}_D{d}"] = {"mean": float(np.mean(c)), "max": int(np.max(c)),
                                           "seed_postings_per_row": sp_mean, "seed_postings_share_of_P": sp_mean * n / P}
    print(f"{kind} data, {n} names, {len(rows)} rows, tile {T}, K {K}; P = {P:.3g} postings")
    print(f"  today   : {out['today_mean']:.1f} candidates per row (max {out['today_max']})")
    print(f"  perfect : {out['perfect_mean']:.1f}")
    for key, v in out["seeded"].items():
        print(f"  seeded {key:10s}: {v['mean']:.1f} (max {v['max']}); seed pass reads {v['seed_postings_per_row']:.0f} postings per row, "
              f"{100 * v['seed_postings_share_of_P']:.2f} % of P")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
