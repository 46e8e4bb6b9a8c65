"""Developer tool: time the top-k epilogue of K3 / K3b on the real movie titles (Netflix 6 172 x IMDB 80 852, the c3 grid) for
ratio, norm_lev, WRatio and jaro_winkler at top_n = 1 (the arg-best path), 5, 10 and 32.

    python tools/k3_topn_time.py [--runs 11] [--warmup 2] [--json OUT] [--profile]

K3 metrics: the lists are staged once (EditQueries / EditTargets); a timed call is edit_argbest_staged (top_n = 1) or
edit_topk_staged, bracketed by CUDA events.  WRatio (K3b) stages its token layouts inside every call, so its events bracket
the whole fuzz_argbest / fuzz_topk call, host staging included.  Per scorer, the top_n values alternate call by call after
warm-up (top_n = 1 next to 10 in every round) and the median of --runs calls is reported.  --profile adds a torch.profiler
table of the device kernels of one top_n = 1 and one top_n = 10 call per scorer."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

SCORERS = ("ratio", "norm_lev", "WRatio", "jaro_winkler")
TOP_NS = (1, 10, 5, 32)


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
    ap.add_argument("--json", default=None)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("k3_topn_time.py needs a CUDA device")
    from polyfuzz_b200 import datasets, editdist, fuzzy

    titles, kind = datasets.load_movie_titles()
    frm, to = titles["Netflix"], titles["IMDB"]
    Q = editdist.EditQueries(frm); T = editdist.EditTargets(to)

    def call(scorer, k):
        if scorer == "WRatio":
            return fuzzy.fuzz_argbest(frm, to, scorer) if k == 1 else fuzzy.fuzz_topk(frm, to, k, scorer)
        return editdist.edit_argbest_staged(Q, T, scorer) if k == 1 else editdist.edit_topk_staged(Q, T, k, scorer)

    out = {"card_before": card(), "data": kind, "n_from": len(frm), "n_to": len(to), "runs": args.runs}
    for scorer in SCORERS:
        for _ in range(args.warmup):
            for k in TOP_NS:
                call(scorer, k)
        torch.cuda.synchronize()
        times = {k: [] for k in TOP_NS}
        for _ in range(args.runs):
            for k in TOP_NS:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                call(scorer, k)
                b.record()
                b.synchronize()
                times[k].append(a.elapsed_time(b))
        res = {}
        for k in TOP_NS:
            t = float(np.median(times[k]))
            res[k] = {"ms": t, "ms_each": [round(x, 3) for x in times[k]], "spread_ms": float(np.max(times[k]) - np.min(times[k]))}
        base = res[1]["ms"]
        print(f"{scorer:13s} " + "  ".join(f"top{k}: {res[k]['ms']:8.3f} ms ({res[k]['ms'] / base:5.3f}x)" for k in sorted(TOP_NS)))
        out[scorer] = {str(k): v for k, v in res.items()}
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for scorer in SCORERS:
            for k in (1, 10):
                call(scorer, k); torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    call(scorer, k); torch.cuda.synchronize()
                print(f"--- {scorer} top_n={k}")
                print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=6))
    out["card_after"] = card()
    print(f"card (name, power limit, SM clock, max SM clock) before: {out['card_before']}\nafter: {out['card_after']}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
