"""Developer tool: time the OSA mode of K3 (normalised optimal string alignment) against normalised Levenshtein and fuzz.ratio on
the real movie titles (Netflix 6 172 x IMDB 80 852, per-row best match), and check a 300-row sample of its arg-best against the
CPU oracle.

    python tools/osa_time.py [--runs 15] [--warmup 3] [--sample 300] [--json OUT]

The lists are staged once (EditQueries / EditTargets); each timed call is edit_argbest_staged (to-list packing per alphabet
batch, the kernels, the split merge), bracketed by CUDA events.  The three metrics alternate call by call after warm-up; the
median and the min-max of --runs calls are reported, with the card's name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

METRICS = ("norm_osa", "norm_lev", "ratio")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv"],
                           capture_output=True, text=True)
        return r.stdout.strip() or r.stderr.strip()
    except OSError as e:
        return f"nvidia-smi not available: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=300)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("osa_time.py needs a CUDA device")
    import osa_oracle
    from polyfuzz_b200 import datasets, editdist

    titles, kind = datasets.load_movie_titles()
    frm, to = titles["Netflix"], titles["IMDB"]
    Q = editdist.EditQueries(frm); T = editdist.EditTargets(to)
    pairs = float(len(frm)) * len(to)
    out = {"card_before": card(), "data": kind, "n_from": len(frm), "n_to": len(to), "pairs": pairs, "runs": args.runs}
    for _ in range(args.warmup):
        for m in METRICS:
            editdist.edit_argbest_staged(Q, T, m)
    torch.cuda.synchronize()
    times = {m: [] for m in METRICS}
    for _ in range(args.runs):
        for m in METRICS:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            editdist.edit_argbest_staged(Q, T, m)
            b.record()
            b.synchronize()
            times[m].append(a.elapsed_time(b))
    out["card_after"] = card()
    for m in METRICS:
        t = float(np.median(times[m]))
        out[m] = {"ms": t, "min_ms": float(min(times[m])), "max_ms": float(max(times[m])), "ms_each": [round(x, 3) for x in times[m]],
                  "pairs_per_s": pairs / (t * 1e-3)}
        print(f"{m:9s} median {t:8.3f} ms  (min {min(times[m]):.3f}, max {max(times[m]):.3f})  pairs/s {pairs / (t * 1e-3):.3e}")
    out["osa_over_lev"] = out["norm_osa"]["ms"] / out["norm_lev"]["ms"]
    print(f"norm_osa / norm_lev: {out['osa_over_lev']:.3f}")

    rng = np.random.default_rng(0)
    rows = np.sort(rng.choice(len(frm), min(args.sample, len(frm)), replace=False))
    sub = [frm[i] for i in rows]
    bi, bs, bd = editdist.edit_argbest(sub, to, "norm_osa")
    oi, os_, od = osa_oracle.osa_argbest(sub, to, "norm_osa", n_threads=os.cpu_count() or 1)
    ok = (np.array_equal(bi.cpu().numpy(), oi) and np.array_equal(bs.cpu().numpy(), os_) and np.array_equal(bd.cpu().numpy(), od))
    out["oracle_check"] = {"rows": len(sub), "equal": bool(ok)}
    print(f"card (before / after timing):\n{out['card_before']}\n{out['card_after']}")
    print(f"oracle check ({len(sub)} rows x {len(to)}, norm_osa): {'equal' if ok else 'DIFFERENT'}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
