"""Developer tool: time weighted Levenshtein (K3 wlev_kernel) on the real movie titles (Netflix 6 172 x IMDB 80 852), per-row best
match and top-10, at weights (1, 1, 1) (the norm_lev path), (1, 1, 2) (the Indel form), (1, 2, 1) and (2, 1, 3) (the bounds and
the queued exact DP); check a sample of every variant's arg-best against the CPU oracle.

    python tools/wlev_time.py [--runs 11] [--warmup 2] [--sample 100] [--json OUT]

The lists are staged once (EditQueries / EditTargets); each timed call is edit_wlev_argbest_staged / edit_wlev_topk_staged
(to-list packing per alphabet batch, the kernels, the split merges), bracketed by CUDA events.  The variants alternate call by
call after warm-up; the median and the min-max of --runs calls are reported, with the card's name, power limit and SM clock read
in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

WEIGHTS = [(1, 1, 1), (1, 1, 2), (1, 2, 1), (2, 1, 3)]


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv"],
                           capture_output=True, text=True)
        return r.stdout.strip() or r.stderr.strip()
    except OSError as e:
        return f"nvidia-smi not available: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=11)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=100)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("wlev_time.py needs a CUDA device")
    import wlev_oracle
    from polyfuzz_b200 import datasets, editdist

    titles, kind = datasets.load_movie_titles()
    frm, to = titles["Netflix"], titles["IMDB"]
    Q = editdist.EditQueries(frm); T = editdist.EditTargets(to)
    variants = {}
    for w in WEIGHTS:
        variants[f"{w} top1"] = lambda w=w: editdist.edit_wlev_argbest_staged(Q, T, w)
        variants[f"{w} top10"] = lambda w=w: editdist.edit_wlev_topk_staged(Q, T, 10, w)
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
        print(f"{name:24s} median {t:9.3f} ms  (min {min(ts):.3f}, max {max(ts):.3f})")

    rng = np.random.default_rng(0)
    rows = np.sort(rng.choice(len(frm), min(args.sample, len(frm)), replace=False))
    sub = [frm[i] for i in rows]
    ok = True
    for w in WEIGHTS:
        bi, bs, bd = editdist.edit_wlev_argbest(sub, to, w)
        oi, os_, od = wlev_oracle.wlev_argbest(sub, to, w, n_threads=os.cpu_count() or 1)
        ok &= bool(np.array_equal(bi.cpu().numpy(), oi) and np.array_equal(bs.cpu().numpy(), os_)
                   and np.array_equal(bd.cpu().numpy(), od))
    out["oracle_check"] = {"rows": len(sub), "weights": WEIGHTS, "equal": ok}
    print(f"card (before / after timing):\n{out['card_before']}\n{out['card_after']}")
    print(f"oracle check ({len(sub)} rows x {len(to)}, every weight triple): {'equal' if ok else 'DIFFERENT'}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
