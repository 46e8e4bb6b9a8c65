"""Candidate mode against all pairs: time and recall of RapidFuzz-style scoring restricted to TF-IDF's top-c candidates.

    python tools/cand_time.py [--out DIR] [--reps N] [--skip-company-all-pairs]

Workloads: the movie titles (6 172 x 80 852, Netflix -> IMDB) and the company names (100 000, self-match), real data from
tests/golden/data when present.  For ratio (K3) and WRatio (K3b) it times, each ending in a device synchronise:
  * all pairs: editdist.edit_argbest / fuzzy.fuzz_argbest (host packing + H2D + kernels), the best to-string per row;
  * TF-IDF: TFIDF(top_n=c, min_similarity=0).match_arrays (K1 + K2) for c in 10, 50, 200;
  * candidate scoring: editdist.edit_cand_topk / fuzzy.fuzz_cand_topk with k = 1 over those candidates.
Recall is the share of rows (with an all-pairs best) whose all-pairs best to-index is among the candidates; "score recall"
counts a row whose candidate best has the all-pairs best score (a tie at another index) as found too.  The card's name and
power limit are read in the same run and written beside the numbers (JSON lines, to stdout and DIR/cand_time.jsonl)."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from polyfuzz_b200 import TFIDF, datasets, editdist, fuzzy  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def timed(fn, reps):
    """(median seconds, last result) of fn() over reps runs, each ended by a device synchronise."""
    ts, out = [], None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), out


def all_pairs(scorer, frm, to):
    self_match = to is frm
    if scorer == "ratio":
        return editdist.edit_argbest(frm, to, "ratio", 0.0, exclude_self=self_match)[:2]
    return fuzzy.fuzz_argbest(frm, to, scorer, 0.0, exclude_self=self_match)


def cand_scoring(scorer, frm, to, cand):
    self_match = to is frm
    if scorer == "ratio":
        return editdist.edit_cand_topk(frm, to, cand, 1, "ratio", 0.0, exclude_self=self_match)[:2]
    return fuzzy.fuzz_cand_topk(frm, to, cand, 1, scorer, 0.0, exclude_self=self_match)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-company-all-pairs", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "cand_time.py measures on the GPU"
    torch.cuda.set_device(0)
    dev = card()
    titles, kt = datasets.load_movie_titles()
    names, kc = datasets.load_company_names(100_000)
    loads = [("titles", kt, titles["Netflix"], titles["IMDB"]), ("company_self", kc, names, names)]
    lines = []

    def emit(rec):
        rec["device"] = dev
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    for name, kind, frm, to in loads:
        to_arg = None if to is frm else to
        for scorer in ("ratio", "WRatio"):
            best = None
            if not (name == "company_self" and args.skip_company_all_pairs):
                all_pairs(scorer, frm[:2000], to)                         # warm-up: modules, staging paths
                reps = args.reps if name == "titles" else 1
                t_all, (bi, bs) = timed(lambda: all_pairs(scorer, frm, to), reps)
                best = (bi.cpu().numpy(), bs.cpu().numpy())
                emit({"workload": name, "data": kind, "n_from": len(frm), "n_to": len(to), "scorer": scorer, "mode": "all_pairs",
                      "ms": round(t_all * 1e3, 2), "reps": reps})
            for c in (10, 50, 200):
                tf = TFIDF(top_n=c, min_similarity=0)
                tf.match_arrays(frm, to_arg)                             # warm-up
                t_tf, (cand, _, _) = timed(lambda: tf.match_arrays(frm, to_arg), args.reps)
                cand_scoring(scorer, frm, to, cand)
                t_sc, (ci, cs) = timed(lambda: cand_scoring(scorer, frm, to, cand), args.reps)
                rec = {"workload": name, "data": kind, "n_from": len(frm), "n_to": len(to), "scorer": scorer, "mode": "candidates",
                       "c": c, "tfidf_ms": round(t_tf * 1e3, 2), "score_ms": round(t_sc * 1e3, 2),
                       "total_ms": round((t_tf + t_sc) * 1e3, 2), "pairs_scored": int((cand >= 0).sum().item())}
                if best is not None:
                    bi, bs = best
                    h = cand.cpu().numpy()
                    has = bi >= 0
                    found = (h[has] == bi[has][:, None]).any(axis=1)
                    same_score = ci.cpu().numpy()[has] >= 0
                    same_score &= cs.cpu().numpy()[has] == bs[has]
                    rec.update(recall=round(float(found.mean()), 4), score_recall=round(float(same_score.mean()), 4),
                               rows_with_best=int(has.sum()))
                emit(rec)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "cand_time.jsonl"), "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
