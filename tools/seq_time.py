"""Developer tool: time K3's sequence metrics (Indel, LCSseq, Hamming, Prefix, Postfix) on the real movie titles (Netflix 6 172 x
IMDB 80 852), per-row best match and top-10, beside norm_lev and ratio; check a sample of every metric's arg-best and top-10
against the plain-Python oracle (tests/seq_oracle.py).

    python tools/seq_time.py [--runs 11] [--warmup 2] [--sample 60] [--json OUT]

The lists are staged once (EditQueries / EditTargets); each timed call is edit_argbest_staged / edit_topk_staged (to-list
packing per alphabet batch, the kernels, the split merges), bracketed by CUDA events.  The variants alternate call by call after
warm-up; the median and the min-max of --runs calls are reported, with the card's name, power limit and SM clock read in the
same run.  The oracle runs first, on the CPU, over --sample rows in parallel processes."""
import argparse
import json
import multiprocessing as mp
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import seq_oracle  # noqa: E402

METRICS = ("norm_lev", "ratio") + seq_oracle.METRICS


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv"],
                           capture_output=True, text=True)
        return r.stdout.strip() or r.stderr.strip()
    except OSError as e:
        return f"nvidia-smi not available: {e}"


def _oracle_row(args):
    """One from-row against the to-list: per sequence metric its top-10 (idx, score, dist) under cutoff 0.0."""
    a, to = args
    lcs = seq_oracle.lcs_matrix([a], to)
    out = {}
    for metric in seq_oracle.METRICS:
        D, _, S = seq_oracle.matrices(metric, [a], to, lcs)
        out[metric] = seq_oracle.topk_from(S, D, 10)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=11)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=60)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from polyfuzz_b200 import datasets

    titles, kind = datasets.load_movie_titles()
    frm, to = titles["Netflix"], titles["IMDB"]
    rng = np.random.default_rng(0)
    rows = np.sort(rng.choice(len(frm), min(args.sample, len(frm)), replace=False))
    sub = [frm[i] for i in rows]
    with mp.get_context("fork").Pool(os.cpu_count() or 1) as pool:        # before CUDA is initialised in this process
        per_row = pool.map(_oracle_row, [(a, to) for a in sub])

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("seq_time.py needs a CUDA device")
    from polyfuzz_b200 import editdist
    Q = editdist.EditQueries(frm); T = editdist.EditTargets(to)
    variants = {}
    for mt in METRICS:
        variants[f"{mt} top1"] = lambda mt=mt: editdist.edit_argbest_staged(Q, T, mt)
        variants[f"{mt} top10"] = lambda mt=mt: editdist.edit_topk_staged(Q, T, 10, mt)
    out = {"card_before": card(), "data": kind, "n_from": len(frm), "n_to": len(to), "pairs": float(len(frm)) * len(to),
           "runs": args.runs}
    for _ in range(args.warmup):
        for f in variants.values():
            f()
    torch.cuda.synchronize()
    times = {name: [] for name in variants}
    for _ in range(args.runs):
        for name, f in variants.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b))
    out["card_after"] = card()
    for name, ts in times.items():
        t = float(np.median(ts))
        out[name] = {"ms": t, "min_ms": float(min(ts)), "max_ms": float(max(ts)), "ms_each": [round(x, 3) for x in ts]}
        print(f"{name:22s} median {t:9.3f} ms  (min {min(ts):.3f}, max {max(ts):.3f})")

    Qs = editdist.EditQueries(sub)
    ok = True
    for metric in seq_oracle.METRICS:
        oi, os_, od = (np.stack([r[metric][c][0] for r in per_row]) for c in range(3))
        bi, bs, bd = editdist.edit_argbest_staged(Qs, T, metric)
        ti, tv = editdist.edit_topk_staged(Qs, T, 10, metric)
        same = (np.array_equal(bi.cpu().numpy(), oi[:, 0]) and np.array_equal(bs.cpu().numpy(), os_[:, 0])
                and np.array_equal(bd.cpu().numpy(), od[:, 0]) and np.array_equal(ti.cpu().numpy(), oi)
                and np.array_equal(tv.cpu().numpy(), os_))
        print(f"oracle check {metric:13s} ({len(sub)} rows x {len(to)}, arg-best and top-10): {'equal' if same else 'DIFFERENT'}")
        ok &= same
    out["oracle_check"] = {"rows": len(sub), "metrics": list(seq_oracle.METRICS), "equal": ok}
    print(f"card (before / after timing):\n{out['card_before']}\n{out['card_after']}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
