"""Developer tool: time unrestricted Damerau-Levenshtein (K3 dl_kernel) on the real movie titles (Netflix 6 172 x IMDB 80 852),
per-row best match and top-10, next to normalised OSA and Levenshtein in the same run, with and without the OSA gate pass; time
the un-gated exact DP (matrix mode) on a slice; check a sample of the arg-best against the CPU oracle.

    python tools/dl_time.py [--runs 11] [--warmup 2] [--slice 200] [--sample 200] [--json OUT]

The lists are staged once (EditQueries / EditTargets); each timed call is edit_argbest_staged / edit_topk_staged (to-list packing
per alphabet batch, the kernels, the split merges), bracketed by CUDA events.  The variants alternate call by call after warm-up;
the median and the min-max of --runs calls are reported, with the card's name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402


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
    ap.add_argument("--slice", type=int, default=200, help="from-rows of the matrix-mode (un-gated DP) timing")
    ap.add_argument("--sample", type=int, default=200)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dl_time.py needs a CUDA device")
    import dl_oracle
    from polyfuzz_b200 import datasets, editdist

    titles, kind = datasets.load_movie_titles()
    frm, to = titles["Netflix"], titles["IMDB"]
    Q = editdist.EditQueries(frm); T = editdist.EditTargets(to)
    Qs = editdist.EditQueries(frm[:args.slice])
    pairs = float(len(frm)) * len(to)
    variants = {
        "norm_dl top1 gated": lambda: editdist.edit_argbest_staged(Q, T, "norm_dl"),
        "norm_dl top1 no gate": lambda: editdist.edit_argbest_staged(Q, T, "norm_dl", dl_gate=False),
        "norm_osa top1": lambda: editdist.edit_argbest_staged(Q, T, "norm_osa"),
        "norm_lev top1": lambda: editdist.edit_argbest_staged(Q, T, "norm_lev"),
        "norm_dl top10 gated": lambda: editdist.edit_topk_staged(Q, T, 10, "norm_dl"),
        "norm_dl top10 no gate": lambda: editdist.edit_topk_staged(Q, T, 10, "norm_dl", dl_gate=False),
        "norm_osa top10": lambda: editdist.edit_topk_staged(Q, T, 10, "norm_osa"),
        "norm_lev top10": lambda: editdist.edit_topk_staged(Q, T, 10, "norm_lev"),
        f"dl matrix {args.slice} rows (DP on every pair)": lambda: editdist.edit_argbest_staged(Qs, T, "dl", want_matrix=True),
    }
    out = {"card_before": card(), "data": kind, "n_from": len(frm), "n_to": len(to), "pairs": pairs, "runs": args.runs}
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
        print(f"{name:44s} median {t:9.3f} ms  (min {min(ts):.3f}, max {max(ts):.3f})")

    rng = np.random.default_rng(0)
    rows = np.sort(rng.choice(len(frm), min(args.sample, len(frm)), replace=False))
    sub = [frm[i] for i in rows]
    bi, bs, bd = editdist.edit_argbest(sub, to, "norm_dl")
    oi, os_, od = dl_oracle.dl_argbest(sub, to, "norm_dl", n_threads=os.cpu_count() or 1)
    ok = (np.array_equal(bi.cpu().numpy(), oi) and np.array_equal(bs.cpu().numpy(), os_) and np.array_equal(bd.cpu().numpy(), od))
    # gated and un-gated calls must agree on the whole grid
    g = editdist.edit_topk_staged(Q, T, 10, "norm_dl"); u = editdist.edit_topk_staged(Q, T, 10, "norm_dl", dl_gate=False)
    same = bool(torch.equal(g[0], u[0]) and torch.equal(g[1], u[1]))
    out["oracle_check"] = {"rows": len(sub), "equal": bool(ok), "gated_equals_ungated_top10": same}
    print(f"card (before / after timing):\n{out['card_before']}\n{out['card_after']}")
    print(f"oracle check ({len(sub)} rows x {len(to)}, norm_dl): {'equal' if ok else 'DIFFERENT'}; "
          f"gated == un-gated top-10: {same}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    if not (ok and same):
        raise SystemExit(1)


if __name__ == "__main__":
    main()
